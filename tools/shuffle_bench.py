"""Cost of the shuffle argument on the GPU prover (one H100).

1. The bench circuit family at 2^20 gates with a shuffle (plonkathon_b200.synthetic.build_circuit(..., shuffle=True),
   two public inputs: a quarter of the rows are in-rows, a quarter out-rows) proved without the shuffle selectors and
   with them.  The witness and every other column are the same, so the difference is the argument: the grand product
   Z3 and its commitment (in the same MSM pass as Z), one coset extension, the quotient's two terms, two evaluations
   and three more round-5 terms.
2. The same comparison with four next-row custom gate terms (992-byte proofs against 864-byte ones).
3. The device memory pb200_prover_set_shuffle adds: Q_in and Q_out three ways (Lagrange, coefficients, 4n coset) and
   Z3 three ways, 18 n field elements by count.

In each comparison the provers alternate after --warmup proofs each; ms per proof is the median of --steps timed proofs
(prove_arrays, host-resident wires).  Every shuffle proof is checked with verify_proof.  The card's name and power limit
are read in the same call.  Prints one JSON object; --out also writes it to a file.

    python tools/shuffle_bench.py --steps 5 --warmup 2 --out profiles/h100_shuffle.json
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
    c = syn.build_circuit(LOG_N, seed=7, n_public=2, custom=terms, shuffle=True)
    pk, *w = syn.circuit_arrays(c)
    custom, shuffle = syn.custom_arrays(c), syn.shuffle_arrays(c)
    plain = pb.Prover.from_arrays(setup, n, pk, custom=custom)
    sh = pb.Prover.from_arrays(setup, n, pk, custom=custom)
    _, mem = alloc(setup, lambda: sh._set_shuffle(*shuffle))
    vk = setup.verification_key_arrays(n, pk, custom=custom, shuffle=shuffle)
    cls = pb.NextRowShuffleProof if terms else pb.ShuffleProof
    public = c.public_values()
    ok = []

    def check(k, raw):
        if k == "shuffle":
            ok.append(vk.verify_proof(n, cls.from_bytes(raw), public))
    t = _time({"without_shuffle": plain, "shuffle": sh}, {"without_shuffle": w, "shuffle": w}, a.steps, a.warmup, check)
    out = {"rows_in": sum(shuffle[0]), "rows_out": sum(shuffle[1]), **t,
           "shuffle_overhead_percent": round(100 * (t["shuffle"]["ms_per_proof"] / t["without_shuffle"]["ms_per_proof"]
                                                    - 1), 2),
           "set_shuffle_memory_MiB": {"measured": round(mem / 2 ** 20, 1), "by_count": round(18 * n * 32 / 2 ** 20, 1)},
           "shuffle_proofs_verified": len(ok) > 0 and all(ok)}
    if terms:
        out["next_row_terms"] = [list(e) for e in terms]
    del plain, sh
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
    setup = pb.Setup.generate(TAU, 1 << LOG_N)
    res["bench_circuit_2p20"] = bench(a, setup, [])
    res["bench_circuit_2p20_four_next_row_terms"] = bench(a, setup, NEXT_TERMS)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
