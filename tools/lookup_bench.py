"""Cost of the lookup argument on the GPU prover (one H100).

1. The bench circuit family at 2^20 gates (plonkathon_b200.synthetic.build_circuit, two public inputs), without and
   with a lookup argument: ``lookup=`` mixes lookup rows into the chain as a fourth kind of row (about a quarter of the
   rows), into a range table of 2^16 rows.  The two provers alternate after --warmup proofs each; ms per proof is the
   median of --steps timed proofs (prove_arrays, host-resident wires).  Memory is the drop in free device memory over
   each Prover.from_arrays (the plain prover is created first, so it also carries the context's one-time tables).
2. 2^16 random 16-bit values, each range-checked, in two circuits, each at the smallest power of two that holds it:
   by lookup, one row per value (a = value, q_K = 1) against the table (v, 0, 0), v < 2^16, and one plain gate
   (2^16 + 1 rows, so 2^17); by bit
   decomposition, 32 rows per value: 16 booleanity gates b (b - 1) = 0 and 16 accumulation gates
   acc' = acc + 2^k b whose last output is the value (2^21 rows).

Every lookup proof is checked with verify_proof.  Prints one JSON object; --out also writes it to a file.

    python tools/lookup_bench.py --steps 5 --warmup 2 --out profiles/h100_lookup.json
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402
from plonkathon_b200.field import CURVE_ORDER as R  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
VALUES, BITS = 1 << 16, 16


def _le(ints):
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in ints), dtype=np.uint8).reshape(-1, 32).copy()


def _small_le(vals, n):
    """small non-negative ints (numpy int64, < 2^63) -> (n,32) uint8, zero padded"""
    out = np.zeros((n, 32), np.uint8)
    out[:len(vals), :8] = np.asarray(vals, dtype="<u8").view(np.uint8).reshape(-1, 8)
    return out


def _time(provers, inputs, steps, warmup, check=None):
    times = {k: [] for k in provers}
    for step in range(warmup + steps):
        for k, prover in provers.items():
            t = time.perf_counter()
            raw = prover.prove_arrays(*inputs[k])
            ms = (time.perf_counter() - t) * 1e3
            if check:
                check(k, raw)
            if step >= warmup:
                times[k].append(ms)
    return {k: {"ms_per_proof": round(statistics.median(v), 2), "ms_min": round(min(v), 2), "ms_max": round(max(v), 2)}
            for k, v in times.items()}


def alloc(setup, fn):
    setup.ctx.sync()
    free0 = torch.cuda.mem_get_info()[0]
    out = fn()
    setup.ctx.sync()
    return out, free0 - torch.cuda.mem_get_info()[0]


def bench_circuit(a, res):
    log_n = 20
    table = [list(range(1 << 16)), [0] * (1 << 16), [0] * (1 << 16)]
    plain_c = syn.build_circuit(log_n, seed=7, n_public=2)
    lk_c = syn.build_circuit(log_n, seed=7, n_public=2, lookup=table)
    n = 1 << log_n
    setup = pb.Setup.generate(TAU, n)
    pk0, *w0 = syn.circuit_arrays(plain_c)
    pk1, *w1 = syn.circuit_arrays(lk_c)
    plain, mem0 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk0))
    lk, mem1 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk1, lookup=syn.lookup_arrays(lk_c)))
    vk = setup.verification_key_arrays(n, pk1, lookup=syn.lookup_arrays(lk_c))
    ok = []
    t = _time({"plain": plain, "lookup": lk}, {"plain": w0, "lookup": w1}, a.steps, a.warmup,
              lambda k, raw: ok.append(vk.verify_proof(n, pb.LookupProof.from_bytes(raw), [int(x) for x in w1[3]]))
              if k == "lookup" else None)
    res["bench_circuit_2p20"] = {
        "lookup_rows": int(sum(lk_c.lookup[0])), "table_rows": 1 << 16, **t,
        "lookup_overhead_percent": round(100 * (t["lookup"]["ms_per_proof"] / t["plain"]["ms_per_proof"] - 1), 2),
        "memory_MiB": {"plain_prover_first": round(mem0 / 2 ** 20, 1), "lookup_prover_second": round(mem1 / 2 ** 20, 1)},
        "lookup_proofs_verified": all(ok)}
    del plain, lk, setup


def range_by_lookup(vals, bits=BITS):
    """one row per value (a = value, b and c unused, q_K = 1, every gate selector 0) against the table (v, 0, 0),
    v < 2^bits, then one gate 1 * 1 = 1: without it the b and c columns would be zero and commit to the identity,
    which the transcript cannot absorb.  2^16 + 1 rows, so 2^17."""
    m = len(vals) + 1
    n = 1 << (m - 1).bit_length()
    none = np.full(n, -1, dtype=np.int64)
    wL, wR, wO = np.arange(n, dtype=np.int64), none.copy(), none.copy()
    wL[m:] = -1
    wR[m - 1], wO[m - 1] = m, m + 1
    S = syn.permutation_polys(wL, wR, wO, n, m)
    zero = np.zeros((n, 32), np.uint8)
    one = np.zeros(n, np.int64)
    one[m - 1] = 1
    QO = [0] * n
    QO[m - 1] = R - 1
    pk = {"QM": _small_le(one, n), "QL": zero, "QR": zero, "QO": _le(QO), "QC": zero,
          "S1": _le(S[0]), "S2": _le(S[1]), "S3": _le(S[2])}
    zcol = np.zeros(1 << bits, np.int64)
    table = (_small_le(np.arange(1 << bits), 1 << bits), _small_le(zcol, 1 << bits), _small_le(zcol, 1 << bits))
    qk = np.zeros(n, np.int64)
    qk[:len(vals)] = 1
    a = np.zeros(n, np.int64)
    a[:len(vals)] = vals
    a[m - 1] = 1
    return n, pk, (_small_le(a, n), _small_le(one, n), _small_le(one, n), []), (_small_le(qk, n), table)


def range_by_bits(vals):
    """32 rows per value: rows 2k (booleanity of bit k: L = R = b, QM = 1, QL = -1) and 2k + 1 (accumulation:
    acc_k+1 = acc_k + 2^k b with L = acc_k, R = b, O = acc_k+1, QL = 1, QR = 2^k, QO = -1; acc_0 is the unused cell)"""
    m = len(vals) * 2 * BITS
    n = 1 << (m - 1).bit_length()
    bits = ((np.asarray(vals)[:, None] >> np.arange(BITS)) & 1).astype(np.int64)      # (values, 16)
    acc = np.cumsum(bits << np.arange(BITS), axis=1)                                  # acc_1 .. acc_16
    nv = len(vals)
    bid = np.arange(nv * BITS, dtype=np.int64).reshape(nv, BITS)                     # variable ids of the bits
    aid = nv * BITS + np.arange(nv * BITS, dtype=np.int64).reshape(nv, BITS)         # of acc_1 .. acc_16
    wL, wR, wO = (np.full(n, -1, np.int64) for _ in range(3))
    QM, QL, QR, QO = (np.zeros(n, dtype=object) for _ in range(4))
    r0 = (np.arange(nv)[:, None] * 2 * BITS + 2 * np.arange(BITS)).reshape(-1)       # booleanity rows
    r1 = r0 + 1
    wL[r0], wR[r0] = bid.reshape(-1), bid.reshape(-1)
    QM[r0], QL[r0] = 1, R - 1
    prev = np.concatenate([np.full((nv, 1), -1), aid[:, :-1]], axis=1).reshape(-1)
    wL[r1], wR[r1], wO[r1] = prev, bid.reshape(-1), aid.reshape(-1)
    QL[r1], QO[r1] = 1, R - 1
    QR[r1] = np.tile(np.array([1 << k for k in range(BITS)], dtype=object), nv)
    S = syn.permutation_polys(wL, wR, wO, n, m)
    values = np.concatenate([bits.reshape(-1), acc.reshape(-1)])

    def col(ids):
        v = np.where(ids >= 0, values[np.maximum(ids, 0)], 0)
        return _small_le(v, n)
    zero = np.zeros((n, 32), np.uint8)
    pk = {"QM": _le(QM), "QL": _le(QL), "QR": _le(QR), "QO": _le(QO), "QC": zero,
          "S1": _le(S[0]), "S2": _le(S[1]), "S3": _le(S[2])}
    return n, pk, (col(wL), col(wR), col(wO), [])


def bench_range(a, res):
    rng = random.Random(16)
    vals = [rng.randrange(1 << BITS) for _ in range(VALUES)]
    n_lk, pk_lk, w_lk, lookup = range_by_lookup(vals)
    n_bits, pk_bits, w_bits = range_by_bits(vals)
    setup = pb.Setup.generate(TAU, max(n_lk, n_bits))
    lk = pb.Prover.from_arrays(setup, n_lk, pk_lk, lookup=lookup)
    bits = pb.Prover.from_arrays(setup, n_bits, pk_bits)
    vk = setup.verification_key_arrays(n_lk, pk_lk, lookup=lookup)
    ok = []
    t = _time({"lookup": lk, "bits": bits}, {"lookup": w_lk, "bits": w_bits}, a.steps, a.warmup,
              lambda k, raw: ok.append(vk.verify_proof(n_lk, pb.LookupProof.from_bytes(raw), [])) if k == "lookup" else None)
    res["range_check_2p16_values_16_bit"] = {
        "lookup": {"rows": len(vals) + 1, "domain": n_lk, "table_rows": 1 << BITS, **t["lookup"]},
        "bit_decomposition": {"rows": 2 * BITS * len(vals), "domain": n_bits, **t["bits"]},
        "lookup_proofs_verified": all(ok)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    res = {"device": torch.cuda.get_device_name(0), "steps": a.steps, "warmup": a.warmup}
    try:
        res["power_limit_W"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                                               "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit_W"] = None
    bench_circuit(a, res)
    bench_range(a, res)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
