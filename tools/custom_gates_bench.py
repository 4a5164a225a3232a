"""Cost of custom gates on the GPU prover (one H100): ms per proof and the prover's per-circuit memory for

  * the bench circuit family at 2^20 gates (plonkathon_b200.synthetic.build_circuit), with 0 custom terms and with all
    four terms of tests/test_custom_gates.py mixed into its rows;
  * a chain of x^5 S-boxes (Poseidon's non-linear layer), once from multiplication rows only (x^2, x^4, x^5: 3 rows per
    S-box) and once with the custom term x^2 * y (x^2, then (x^2)^2 * x: 2 rows).  The S-box count is chosen so that the
    custom circuit fills 2^20 rows and the plain one needs 2^21.

Proofs run one after another (prove_arrays, host-resident wires); ms per proof is the median of --steps timed proofs after
--warmup, proofs/s is its inverse.  Memory is the drop in free device memory over Prover.from_arrays.  Prints one JSON
object; --out also writes it to a file.

    python tools/custom_gates_bench.py --steps 5 --warmup 2 --out profiles/h100_custom_gates.json
"""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

R = syn.R
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
ALL_TERMS = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]


def sbox_chain(count: int, custom: bool) -> syn.ArrayCircuit:
    """x_0 public, x_(t+1) = x_t^5, ``count`` S-boxes"""
    per = 2 if custom else 3
    m = 1 + per * count
    n = 1 << max(1, (m - 1).bit_length())
    wL, wR, wO = (np.full(n, -1, dtype=np.int64) for _ in range(3))
    QL, QR, QM, QO, QC = ([0] * n for _ in range(5))
    QK = [0] * n
    values = [3]
    wL[0], QL[0] = 0, 1  # public input row
    x, row = 0, 1

    def new(v):
        values.append(v)
        return len(values) - 1

    def mul(a, b):
        nonlocal row
        out = new(values[a] * values[b] % R)
        wL[row], wR[row], wO[row], QM[row], QO[row] = a, b, out, R - 1, 1
        row += 1
        return out

    for _ in range(count):
        x2 = mul(x, x)
        if custom:  # x^5 = (x^2)^2 * x in one row: Q = -1 on the term a^2 b, QO = 1
            out = new(values[x2] * values[x2] % R * values[x] % R)
            wL[row], wR[row], wO[row], QK[row], QO[row] = x2, x, out, R - 1, 1
            row += 1
            x = out
        else:
            x = mul(mul(x2, x2), x)
    terms = [((2, 1, 0), QK)] if custom else []
    return syn.ArrayCircuit(n, m, wL, wR, wO, QL, QR, QM, QO, QC, 1, values, [], terms)


def measure(c: syn.ArrayCircuit, steps: int, warmup: int, setups: dict) -> dict:
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    custom = syn.custom_arrays(c)
    if n not in setups:
        setups.clear()
        torch.cuda.empty_cache()
        setups[n] = pb.Setup.generate(TAU, n)
    setup = setups[n]
    setup.ctx.sync()
    free0 = torch.cuda.mem_get_info()[0]
    prover = pb.Prover.from_arrays(setup, n, pk, custom=custom)
    setup.ctx.sync()
    mem = free0 - torch.cuda.mem_get_info()[0]
    first = None
    for _ in range(warmup):
        first = prover.prove_arrays(A, B, C, public)
    ms = []
    for _ in range(steps):
        t = time.perf_counter()
        raw = prover.prove_arrays(A, B, C, public)
        ms.append((time.perf_counter() - t) * 1e3)
        assert first is None or raw == first
    vk = setup.verification_key_arrays(n, pk, custom=custom)
    ok = vk.verify_proof(n, pb.Proof.from_bytes(raw), public)
    del prover
    med = statistics.median(ms)
    return {"log_n": n.bit_length() - 1, "rows_used": c.n_constraints, "custom_terms": [list(e) for e, _ in c.custom],
            "ms_per_proof": round(med, 2), "ms_min": round(min(ms), 2), "ms_max": round(max(ms), 2),
            "proofs_per_s": round(1e3 / med, 2), "prover_memory_MiB": round(mem / 2 ** 20, 1), "proof_verified": ok}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()
    setups = {}
    res = {"device": torch.cuda.get_device_name(0), "steps": a.steps, "warmup": a.warmup}
    try:
        import subprocess
        res["power_limit_W"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                                               "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit_W"] = None
    res["bench_0_terms"] = measure(syn.build_circuit(a.log_n, n_public=2), a.steps, a.warmup, setups)
    res["bench_4_terms"] = measure(syn.build_circuit(a.log_n, n_public=2, custom=ALL_TERMS), a.steps, a.warmup, setups)
    sboxes = ((1 << a.log_n) - 1) // 2
    res["sbox_count"] = sboxes
    res["sbox_custom_x2y"] = measure(sbox_chain(sboxes, True), a.steps, a.warmup, setups)
    res["sbox_mul_rows_only"] = measure(sbox_chain(sboxes, False), a.steps, a.warmup, setups)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
