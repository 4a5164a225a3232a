"""The witness check (``Prover.check_arrays``, csrc/check.cu) beside one proof of the same circuit, on the bench circuit
family (plonkathon_b200.synthetic.build_circuit, seed 7, two public inputs) at 2^20, 2^22 and 2^24 gates:

  * the first check of a prover, which also builds and keeps sigma, with the wires resident on the device;
  * the median of --reps later checks with the wires on the device (pb200_prover_check_device), so sigma's build is the
    first call less this median, and the median of --reps checks from host arrays (pb200_prover_check, as prove_arrays
    takes them: the 96n bytes of wires cross PCIe in every call);
  * one proof (prove_arrays) after one warm-up proof;
  * the peak device memory of the first and of a later check: sampled, the largest drop of free device memory
    (cudaMemGetInfo, polled every 0.5 ms from a second thread) below what was free before the call, and counted, the
    bytes the call checks against free memory before any device work (DESIGN.md section 2) without cub's storage.

Times are host wall clock around calls that return after their results are on the host.  The card's name and power limit
are read in the same run.  Prints one JSON object; --out also writes it to a file.

    python tools/check_bench.py --out profiles/h100_check.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
MIB = 2 ** 20


def peak_during(fn):
    """(fn's result, seconds, MiB of the largest drop of free device memory while fn ran)"""
    base, _ = torch.cuda.mem_get_info()
    low = [base]
    done = threading.Event()

    def poll():
        while not done.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info()[0])
            time.sleep(0.0005)
    t = threading.Thread(target=poll)
    t.start()
    t0 = time.perf_counter()
    try:
        out = fn()
    finally:
        dt = time.perf_counter() - t0
        done.set()
        t.join()
    return out, dt, (base - low[0]) / MIB


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = {"gpu": gpu, "circuit": "synthetic.build_circuit(log_n, seed=7, n_public=2)", "reps": args.reps, "sizes": {}}
    torch.cuda.init()
    for log_n in [int(x) for x in args.sizes.split(",")]:
        n = 1 << log_n
        t0 = time.time()
        c = syn.build_circuit(log_n, seed=7, n_public=2)
        pk, A, B, C, public = syn.circuit_arrays(c)
        del c
        host_s = time.time() - t0
        setup = pb.Setup.generate(TAU, n)
        prover = pb.Prover.from_arrays(setup, n, pk)
        dev = [torch.from_numpy(x).cuda() for x in (A, B, C)]
        rep, first_s, first_mib = peak_during(lambda: prover.check_arrays(*dev, public))
        assert rep.ok, str(rep)
        times = {"device": [], "host": []}
        later_mib = 0.0
        for _ in range(args.reps):
            for where, wires in (("device", dev), ("host", (A, B, C))):
                rep, dt, mib = peak_during(lambda: prover.check_arrays(*wires, public))
                assert rep.ok
                times[where].append(dt * 1e3)
                later_mib = max(later_mib, mib)
        raw = prover.prove_arrays(A, B, C, public)
        t0 = time.perf_counter()
        assert prover.prove_arrays(A, B, C, public) == raw
        proof_ms = (time.perf_counter() - t0) * 1e3
        dev_ms, host_ms = statistics.median(times["device"]), statistics.median(times["host"])
        m = 3 * n
        res["sizes"]["2^%d" % log_n] = {
            "sliced": prover.sliced, "first_check_ms_device_wires": round(first_s * 1e3, 1),
            "sigma_build_ms": round(first_s * 1e3 - dev_ms, 1), "check_ms_device_wires": round(dev_ms, 1),
            "check_ms_host_wires": round(host_ms, 1), "check_ms_all": {k: [round(t, 1) for t in v] for k, v in times.items()},
            "proof_ms": round(proof_ms, 1), "check_over_proof_device_wires": round(dev_ms / proof_ms, 3),
            "check_over_proof_host_wires": round(host_ms / proof_ms, 3),
            "peak_mib_sampled_first_check": round(first_mib), "peak_mib_sampled_later_check": round(later_mib),
            "peak_mib_counted_first_check": round((m * 56 + 64) / MIB),
            "peak_mib_counted_later_check": round((m * 38 + 64 + 12 * 16) / MIB),
            "sigma_mib": round(12 * n / MIB), "host_circuit_build_s": round(host_s, 1)}
        del dev
        print(json.dumps({"2^%d" % log_n: res["sizes"]["2^%d" % log_n]}), flush=True)
        del prover, setup
        torch.cuda.empty_cache()
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
