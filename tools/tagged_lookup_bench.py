"""Cost of lookups over several tables (a table tag) on the GPU prover (one H100).

The bench circuit family at 2^20 gates (plonkathon_b200.synthetic.build_circuit, two public inputs, seed 7) with a
quarter of its rows as lookups, each row into one of three tables picked at random: a 16-bit range table (v, 0, 0),
a 4-bit XOR table and a 4-bit AND table (2^16 + 512 rows).  Three provers:
  * ``tagged``: ``lookups=`` the three tables (t4 and Q_T, PlonKup's table tag);
  * ``one_table``: the same witness and the same lookup rows against the three tables merged into one untagged table
    (``lookup=``; unsound for XOR beside AND, here only as the cost without the tag);
  * ``plain``: the same seed without lookups.
The provers alternate after --warmup proofs each; ms per proof is the median of --steps timed proofs (prove_arrays,
host-resident wires).  Memory is the drop in free device memory over each Prover.from_arrays (the plain prover is
created first, so it also carries the context's one-time tables).  Every lookup proof is checked with verify_proof.
Prints one JSON object; --out also writes it to a file.

    python tools/tagged_lookup_bench.py --steps 5 --warmup 2 --out profiles/h100_tagged_lookup.json
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
from lookup_bench import TAU, _time, alloc  # noqa: E402


def op_table(bits, op):
    rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(c) for c in zip(*rows)]


def bench(a, res):
    log_n = 20
    n = 1 << log_n
    tables = [[list(range(1 << 16)), [0] * (1 << 16), [0] * (1 << 16)], op_table(4, lambda x, y: x ^ y),
              op_table(4, lambda x, y: x & y)]
    plain_c = syn.build_circuit(log_n, seed=7, n_public=2)
    c = syn.build_circuit(log_n, seed=7, n_public=2, lookups=tables)
    merged = ([int(any(q[i] for q, _ in c.lookups)) for i in range(n)],
              tuple([x for t in tables for x in t[w]] for w in range(3)))
    setup = pb.Setup.generate(TAU, n)
    pk0, *w0 = syn.circuit_arrays(plain_c)
    pk1, *w1 = syn.circuit_arrays(c)
    plain, mem0 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk0))
    one, mem1 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk1, lookup=merged))
    tagged, mem2 = alloc(setup, lambda: pb.Prover.from_arrays(setup, n, pk1, lookups=syn.lookups_arrays(c)))
    vks = {"one_table": setup.verification_key_arrays(n, pk1, lookup=merged),
           "tagged": setup.verification_key_arrays(n, pk1, lookups=syn.lookups_arrays(c))}
    public = [int(x) for x in w1[3]]
    ok = []
    t = _time({"plain": plain, "one_table": one, "tagged": tagged}, {"plain": w0, "one_table": w1, "tagged": w1},
              a.steps, a.warmup,
              lambda k, raw: ok.append(vks[k].verify_proof(n, pb.LookupProof.from_bytes(raw), public))
              if k in vks else None)
    ms = {k: v["ms_per_proof"] for k, v in t.items()}
    res["bench_circuit_2p20_three_tables"] = {
        "lookup_rows_per_table": [int(sum(q)) for q, _ in c.lookups], "table_rows": [len(x[0]) for x in tables], **t,
        "tag_overhead_percent_vs_one_table": round(100 * (ms["tagged"] / ms["one_table"] - 1), 2),
        "memory_MiB": {"plain_prover_first": round(mem0 / 2 ** 20, 1), "one_table_prover": round(mem1 / 2 ** 20, 1),
                       "tagged_prover": round(mem2 / 2 ** 20, 1),
                       "tag_extra": round((mem2 - mem1) / 2 ** 20, 1)},
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
    bench(a, res)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
