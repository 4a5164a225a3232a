"""Large circuits on one GPU: the full round 3 against the sliced one (csrc/memory_plan.cuh, "sliced round 3" in
csrc/prover.cu) on the bench circuit family (plonkathon_b200.synthetic.build_circuit, seed 7, two public inputs).

  * 2^22 and 2^23 gates: a full prover and a sliced one (PB200_SLICED=1), proofs alternating between them, median of
    --reps timed proofs each after one warm-up proof; both must give the same bytes;
  * 2^24 gates: the prover the planner picks without the knob (sliced: the full path does not fit 80 GB), median of
    --reps-2p24 timed proofs after one warm-up proof.

Every prover gets a context of its own (stream, scratch, NTT plans), so the drop in free device memory over its
creation and over its first proof is its own; the planner's count for the same prover stands beside each (the count
of the host self-test library, compiled into a temporary directory).  ms per proof is host wall clock around
prove_arrays (host-resident wires, which returns after the proof is on the host).  The card's name and power limit
are read in the same run.  Prints one JSON object; --out also writes it to a file.

    python tools/large_circuit_bench.py --out profiles/h100_large_circuits.json
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import _lib  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
GIB = 2 ** 30


def planner():
    csrc = os.path.join(ROOT, "plonkathon_b200", "csrc")
    out = os.path.join(tempfile.mkdtemp(prefix="pb200_plan_"), "plan.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++",
                           os.path.join(csrc, "host_selftest.cpp"), "-I", csrc, "-o", out])
    L = ctypes.CDLL(out)
    L.hs_prover_memory.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64,
                                   ctypes.c_uint64, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]

    def predict(log_n):
        """GiB by count: {layout: {creation, total}}; creation leaves out the MSM scratch, which the first proof grows"""
        c = ctypes.c_uint64 * 8
        o = c()
        L.hs_prover_memory(log_n, 0, min(max(log_n, 4), 21), 3, 0, 0, 0, o)
        res = {}
        for k, name in enumerate(("full", "sliced")):
            circuit, proof, ntt, msm = o[4 * k:4 * k + 4]
            res[name] = {"circuit": circuit / GIB, "proof": proof / GIB, "ntt": ntt / GIB, "msm": msm / GIB,
                         "total": (circuit + proof + ntt + msm) / GIB}
        return res
    return predict


def free_gib():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0] / GIB


def make_prover(setup, n, pk, sliced):
    if sliced:
        os.environ["PB200_SLICED"] = "1"
    else:
        os.environ.pop("PB200_SLICED", None)
    ctx = _lib.Context(0)
    f0 = free_gib()
    prover = pb.Prover.from_arrays(setup, n, pk, ctx=ctx)
    os.environ.pop("PB200_SLICED", None)
    return ctx, prover, f0 - free_gib()


def timed(prover, args):
    t = time.perf_counter()
    raw = prover.prove_arrays(*args)
    return raw, (time.perf_counter() - t) * 1e3


def run_size(log_n, reps, predict, modes):
    n = 1 << log_n
    t = time.perf_counter()
    c = syn.build_circuit(log_n, seed=7, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    del c
    build_s = time.perf_counter() - t
    setup = pb.Setup.generate(TAU, n)
    res = {"log_n": log_n, "circuit_build_s": round(build_s, 1), "predicted_GiB": predict(log_n), "modes": {}}
    lanes = {}
    for sliced in modes:
        ctx, prover, created = make_prover(setup, n, pk, sliced)
        f0 = free_gib()
        raw, first_ms = timed(prover, (A, B, C, public))
        name = "sliced" if prover.sliced else "full"
        assert sliced is None or prover.sliced == sliced
        lanes[name] = (ctx, prover)
        res["modes"][name] = {"sliced": prover.sliced, "free_drop_creation_GiB": round(created, 3),
                              "free_drop_first_proof_GiB": round(f0 - free_gib(), 3),
                              "first_proof_ms": round(first_ms, 1), "ms": [], "proof_sha_prefix": raw[:8].hex()}
    proofs = {}
    for _ in range(reps):  # alternating, so both paths see the same state of the shared machine
        for name, (_, prover) in lanes.items():
            raw, ms = timed(prover, (A, B, C, public))
            res["modes"][name]["ms"].append(round(ms, 1))
            proofs.setdefault(name, set()).add(raw)
    for name, m in res["modes"].items():
        m["ms_per_proof"] = round(statistics.median(m["ms"]), 1)
    res["deterministic"] = all(len(v) == 1 for v in proofs.values())
    if len(proofs) == 2:
        res["full_equals_sliced"] = proofs["full"] == proofs["sliced"]
        f, s = res["modes"]["full"]["ms_per_proof"], res["modes"]["sliced"]["ms_per_proof"]
        res["sliced_over_full"] = round(s / f, 3)
    lanes.clear()
    del setup
    torch.cuda.synchronize()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="22,23,24", help="log2 gate counts; 24 runs the planner's own choice only")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--reps-2p24", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    predict = planner()
    res = {"device": torch.cuda.get_device_name(0), "total_GiB": round(torch.cuda.mem_get_info()[1] / GIB, 2)}
    try:
        res["power_limit_W"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["power_limit_W"] = None
    res["sizes"] = []
    for lg in (int(x) for x in a.sizes.split(",")):
        if lg >= 24:
            r = run_size(lg, a.reps_2p24, predict, (None,))
        else:
            r = run_size(lg, a.reps, predict, (False, True))
        res["sizes"].append(r)
        print(json.dumps(r), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
