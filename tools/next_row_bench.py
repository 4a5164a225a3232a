"""Cost of custom gate terms over the next row on the GPU prover (one H100).

1. The bench circuit family at 2^20 gates (plonkathon_b200.synthetic.build_circuit, two public inputs) with four
   next-row terms (a', a a', b'^2 c', b c c') against the same family with four same-row terms (a^2, c^3, a^2 b, a b c).
   The difference is the cost of the shifted reads in the quotient, the three more evaluations of round 4 and the
   three-vector zeta w batch of round 5.
2. 16-bit range checks of as many random values as fit in 2^20 rows at 17 rows per value: by the running sum over the
   next row (synthetic.range_check_circuit, one row per bit, 2^20 rows) against tools/lookup_bench.py's bit
   decomposition of the same values (two rows per bit, which needs 2^21 rows).
3. The two circuits of 1 in zero-knowledge mode (fresh blinders), with and without next-row terms.

In each comparison the provers alternate after --warmup proofs each; ms per proof is the median of --steps timed proofs
(prove_arrays, host-resident wires).  Every next-row proof is checked with verify_proof.  The card's name and power
limit are read in the same call.  Prints one JSON object; --out also writes it to a file.

    python tools/next_row_bench.py --steps 5 --warmup 2 --out profiles/h100_next_row.json
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402
from lookup_bench import _time, alloc, range_by_bits  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
NEXT_TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
SAME_TERMS = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]
LOG_N, BITS = 20, 16


def _verifier(setup, n, pk, c, ok):
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c))
    public = c.public_values()

    def check(k, raw):
        if len(raw) == 864:
            ok.append(vk.verify_proof(n, pb.NextRowProof.from_bytes(raw), public))
    return check


def bench_terms(a, res, setup):
    n = 1 << LOG_N
    nr_c = syn.build_circuit(LOG_N, seed=7, n_public=2, custom=NEXT_TERMS)
    sr_c = syn.build_circuit(LOG_N, seed=7, n_public=2, custom=SAME_TERMS)
    pk0, *w0 = syn.circuit_arrays(sr_c)
    pk1, *w1 = syn.circuit_arrays(nr_c)
    same, mem0 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk0, custom=syn.custom_arrays(sr_c)))
    nxt, mem1 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk1, custom=syn.custom_arrays(nr_c)))
    ok = []
    check = _verifier(setup, n, pk1, nr_c, ok)
    t = _time({"same_row": same, "next_row": nxt}, {"same_row": w0, "next_row": w1}, a.steps, a.warmup, check)
    res["bench_circuit_2p20_four_terms"] = {
        "next_row_terms": [list(e) for e in NEXT_TERMS], "same_row_terms": [list(e) for e in SAME_TERMS],
        "rows_per_term_next_row": [sum(1 for x in col if x) for _, col in nr_c.custom], **t,
        "next_row_overhead_percent": round(100 * (t["next_row"]["ms_per_proof"] / t["same_row"]["ms_per_proof"] - 1), 2),
        "memory_MiB": {"same_row_prover_first": round(mem0 / 2 ** 20, 1), "next_row_prover_second": round(mem1 / 2 ** 20, 1)},
        "next_row_proofs_verified": len(ok) > 0 and all(ok)}
    # 3: the same two provers in zero-knowledge mode
    same.set_zk(True)
    nxt.set_zk(True)
    ok = []
    t = _time({"same_row_zk": same, "next_row_zk": nxt}, {"same_row_zk": w0, "next_row_zk": w1}, a.steps, a.warmup,
              _verifier(setup, n, pk1, nr_c, ok))
    res["zero_knowledge_2p20_four_terms"] = {
        **t, "next_row_overhead_percent": round(100 * (t["next_row_zk"]["ms_per_proof"] /
                                                       t["same_row_zk"]["ms_per_proof"] - 1), 2),
        "next_row_proofs_verified": len(ok) > 0 and all(ok)}
    del same, nxt


def bench_range(a, res, setup):
    n_values = ((1 << LOG_N) - 2) // (BITS + 1)
    rs_c = syn.range_check_circuit(LOG_N, n_values, bits=BITS, seed=16)
    vals = [rs_c.values[i] for i in rs_c.wire_L[(BITS + 1) + 1::BITS + 1][:n_values].tolist()]
    assert len(vals) == n_values
    n_rs = rs_c.group_order
    pk_rs, *w_rs = syn.circuit_arrays(rs_c)
    n_bits, pk_bits, w_bits = range_by_bits(vals)
    rs = pb.Prover.from_arrays(setup, n_rs, pk_rs, custom=syn.custom_arrays(rs_c))
    bits = pb.Prover.from_arrays(setup, n_bits, pk_bits)
    ok = []
    t = _time({"running_sum": rs, "bits": bits}, {"running_sum": w_rs, "bits": w_bits}, a.steps, a.warmup,
              _verifier(setup, n_rs, pk_rs, rs_c, ok))
    res["range_check_16_bit"] = {
        "values": n_values,
        "running_sum": {"rows": rs_c.n_constraints, "domain": n_rs, **t["running_sum"]},
        "bit_decomposition": {"rows": 2 * BITS * n_values, "domain": n_bits, **t["bits"]},
        "running_sum_proofs_verified": len(ok) > 0 and all(ok)}


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
    setup = pb.Setup.generate(TAU, (1 << (LOG_N + 1)))  # the decomposition's 2^21 rows; n + 9 for zero knowledge
    bench_terms(a, res, setup)
    bench_range(a, res, setup)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
