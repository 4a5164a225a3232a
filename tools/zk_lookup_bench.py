"""Cost of zero-knowledge lookup proofs on the GPU prover (one H100).

The bench circuit family at 2^20 gates (plonkathon_b200.synthetic.build_circuit, two public inputs, seed 7) with a
quarter of its rows as lookups into three tables told apart by a table tag: a 16-bit range table (v, 0, 0), a 4-bit XOR
table and a 4-bit AND table.  Two provers of the same circuit and SRS (n + 6 powers):
  * ``lookup``: plain lookup proofs;
  * ``zk_lookup``: the same prover kind after ``set_zk_lookup(True)`` (fresh OS randomness for every proof).
The provers alternate after --warmup proofs each; ms per proof is the median of --steps timed proofs (prove_arrays,
host-resident wires).  Memory: the drop in free device memory over each Prover.from_arrays, and over set_zk_lookup
(the blinded buffers of n + 8 coefficients).  Every proof is checked with verify_proof.  Prints one JSON object; --out
also writes it to a file.

    python tools/zk_lookup_bench.py --steps 5 --warmup 2 --out profiles/h100_zk_lookup.json
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
from tagged_lookup_bench import op_table  # noqa: E402


def bench(a, res):
    log_n = 20
    n = 1 << log_n
    tables = [[list(range(1 << 16)), [0] * (1 << 16), [0] * (1 << 16)], op_table(4, lambda x, y: x ^ y),
              op_table(4, lambda x, y: x & y)]
    c = syn.build_circuit(log_n, seed=7, n_public=2, lookups=tables)
    setup = pb.Setup.generate(TAU, n + 6)
    pk, *w = syn.circuit_arrays(c)
    make = lambda: pb.Prover.from_arrays(setup, n, pk, lookups=syn.lookups_arrays(c))  # noqa: E731
    lk, mem_lk = alloc(setup, make)
    zk, mem_zk_prover = alloc(setup, make)
    _, mem_zk_mode = alloc(setup, lambda: zk.set_zk_lookup(True))
    vk = setup.verification_key_arrays(n, pk, lookups=syn.lookups_arrays(c))
    public = [int(x) for x in w[3]]
    ok = []
    t = _time({"lookup": lk, "zk_lookup": zk}, {"lookup": w, "zk_lookup": w}, a.steps, a.warmup,
              lambda k, raw: ok.append(vk.verify_proof(n, pb.LookupProof.from_bytes(raw), public)))
    ms = {k: v["ms_per_proof"] for k, v in t.items()}
    res["bench_circuit_2p20_three_tables"] = {
        "lookup_rows_per_table": [int(sum(q)) for q, _ in c.lookups], "table_rows": [len(x[0]) for x in tables], **t,
        "zk_overhead_percent": round(100 * (ms["zk_lookup"] / ms["lookup"] - 1), 2),
        "memory_MiB": {"lookup_prover_first": round(mem_lk / 2 ** 20, 1),
                       "second_lookup_prover": round(mem_zk_prover / 2 ** 20, 1),
                       "set_zk_lookup": round(mem_zk_mode / 2 ** 20, 1)},
        "proofs_verified": all(ok)}


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
