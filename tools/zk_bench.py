"""Cost of zero-knowledge proving on the GPU prover (one H100): the bench circuit family at 2^20 gates
(plonkathon_b200.synthetic.build_circuit, two public inputs) proved in plain and in zero-knowledge mode.

One SRS of 2^20 + 6 generated points serves both provers.  The modes alternate (plain, zk, plain, zk, ...) after
--warmup proofs of each; ms per proof is the median of --steps timed proofs per mode (prove_arrays, host-resident wires,
fresh OS randomness for every zero-knowledge proof).  Memory is the drop in free device memory over each
Prover.from_arrays (the first prover of the process also allocates the context's one-time tables) and over set_zk (the
blinded vectors: 7 buffers of n + 8 elements, and round 5's scratch grown to n + 8).  Every plain proof must equal the golden 2^20 proof (tests/golden/proof_2p20.json); every
zero-knowledge proof must verify (verify_proof) and differ from the others.  Prints one JSON object; --out also writes it to a file.

    python tools/zk_bench.py --steps 5 --warmup 2 --out profiles/h100_zk.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out")
    a = ap.parse_args()
    log_n = 20
    rec = json.load(open(os.path.join(ROOT, "tests", "golden", "proof_2p20.json")))
    res = {"device": torch.cuda.get_device_name(0), "steps": a.steps, "warmup": a.warmup, "log_n": log_n}
    try:
        res["power_limit_W"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                                               "-i", "0"], capture_output=True, text=True).stdout.strip()
    except OSError:
        res["power_limit_W"] = None
    c = syn.build_circuit(log_n, seed=rec["seed"], n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n + 6)
    res["srs_points"] = n + 6

    def alloc(fn):
        setup.ctx.sync()
        free0 = torch.cuda.mem_get_info()[0]
        out = fn()
        setup.ctx.sync()
        return out, free0 - torch.cuda.mem_get_info()[0]

    plain, mem_plain = alloc(lambda: pb.Prover.from_arrays(setup, n, pk))
    zk, mem_zk_prover = alloc(lambda: pb.Prover.from_arrays(setup, n, pk))
    _, mem_zk_buffers = alloc(lambda: zk.set_zk(True))
    provers = {"plain": plain, "zk": zk}
    times = {"plain": [], "zk": []}
    zk_proofs = []
    plain_ok = True
    for step in range(a.warmup + a.steps):
        for mode, prover in provers.items():
            t = time.perf_counter()
            raw = prover.prove_arrays(A, B, C, public)
            ms = (time.perf_counter() - t) * 1e3
            if mode == "plain":
                plain_ok &= raw.hex() == rec["proof_hex"]
            else:
                zk_proofs.append(raw)
            if step >= a.warmup:
                times[mode].append(ms)
    vk = setup.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    zk_ok = all(vk.verify_proof(n, pb.Proof.from_bytes(raw), pub) for raw in zk_proofs)
    for mode in ("plain", "zk"):
        ms = times[mode]
        res[mode] = {"ms_per_proof": round(statistics.median(ms), 2), "ms_min": round(min(ms), 2),
                     "ms_max": round(max(ms), 2), "proofs_per_s": round(1e3 / statistics.median(ms), 2)}
    res["zk_overhead_percent"] = round(100 * (res["zk"]["ms_per_proof"] / res["plain"]["ms_per_proof"] - 1), 2)
    res["memory_MiB"] = {"plain_prover_first": round(mem_plain / 2 ** 20, 1),
                         "zk_prover_second": round(mem_zk_prover / 2 ** 20, 1),
                         "set_zk": round(mem_zk_buffers / 2 ** 20, 1)}
    res["plain_proofs_match_golden"] = plain_ok
    res["zk_proofs_distinct"] = len(set(zk_proofs)) == len(zk_proofs)
    res["zk_proofs_verified"] = zk_ok
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
