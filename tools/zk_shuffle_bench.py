"""Cost of zero-knowledge shuffle proofs on the GPU prover (one H100).

The bench circuit family at 2^20 gates with a shuffle (plonkathon_b200.synthetic.build_circuit(..., shuffle=True), two
public inputs, seed 7: a quarter of the rows are in-rows, a quarter out-rows), without and with four next-row custom
gate terms.  Two provers of the same circuit on one SRS of n + 9 powers:
  * ``shuffle``: plain shuffle proofs;
  * ``zk_shuffle``: the same prover kind after ``set_zk_shuffle(True)`` (fresh OS randomness for every proof).
The provers alternate after --warmup proofs each; ms per proof is the median of --steps timed proofs (prove_arrays,
host-resident wires).  Memory: the drop in free device memory over set_zk_shuffle, against the count of zero-knowledge
mode's buffers plus Z3': eight vectors of n + pad elements (A' B' C' Z' Z3' T1' T2' T3', pad = 8, or 9 with next-row
terms), and the five round-5 scratch vectors grown from n to n + pad.  Every proof is checked with verify_proof.  The
card's name and power limit are read in the same call.  Prints one JSON object; --out also writes it to a file.

    python tools/zk_shuffle_bench.py --steps 5 --warmup 2 --out profiles/h100_zk_shuffle.json
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
from lookup_bench import _time, alloc  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
NEXT_TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
LOG_N = 20


def bench(a, setup, terms):
    n = 1 << LOG_N
    pad = 9 if terms else 8
    c = syn.build_circuit(LOG_N, seed=7, n_public=2, custom=terms, shuffle=True)
    pk, *w = syn.circuit_arrays(c)
    custom, shuffle = syn.custom_arrays(c), syn.shuffle_arrays(c)
    make = lambda: pb.Prover.from_arrays(setup, n, pk, custom=custom, shuffle=shuffle)  # noqa: E731
    plain, zk = make(), make()
    _, mem = alloc(setup, lambda: zk.set_zk_shuffle(True))
    vk = setup.verification_key_arrays(n, pk, custom=custom, shuffle=shuffle)
    cls = pb.NextRowShuffleProof if terms else pb.ShuffleProof
    public = c.public_values()
    ok = []
    t = _time({"shuffle": plain, "zk_shuffle": zk}, {"shuffle": w, "zk_shuffle": w}, a.steps, a.warmup,
              lambda k, raw: ok.append(vk.verify_proof(n, cls.from_bytes(raw), public)))
    # A' B' C' Z' Z3', T1' T2' T3' (n + pad each) and the five round-5 scratch vectors grown from n to n + pad
    by_count = (8 * (n + pad) + 5 * pad) * 32
    out = {"rows_in": sum(shuffle[0]), "rows_out": sum(shuffle[1]), **t,
           "zk_overhead_percent": round(100 * (t["zk_shuffle"]["ms_per_proof"] / t["shuffle"]["ms_per_proof"] - 1), 2),
           "set_zk_shuffle_memory_MiB": {"measured": round(mem / 2 ** 20, 1), "by_count": round(by_count / 2 ** 20, 1)},
           "proofs_verified": len(ok) > 0 and all(ok)}
    if terms:
        out["next_row_terms"] = [list(e) for e in terms]
    del plain, zk
    return out


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
    setup = pb.Setup.generate(TAU, (1 << LOG_N) + 9)
    res["bench_circuit_2p20"] = bench(a, setup, [])
    res["bench_circuit_2p20_four_next_row_terms"] = bench(a, setup, NEXT_TERMS)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
