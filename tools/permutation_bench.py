"""The copy-constraint permutation on the GPU (plonkathon_b200.permutation_arrays, csrc/permutation.cu) against its CPU
restatement (synthetic.permutation_polys) on the bench circuit family (synthetic.build_circuit, seed 7, two public
inputs), at 2^20, 2^22 and 2^24 gates by default.

Each circuit is built once, outside every timed region.  Per size:
  * gpu_ms: CUDA events on the context's stream around the whole call (host ids in, S1..S3 back in host memory), after
    one warm-up call; median (and all values) of --reps calls;
  * cpu_s: one run of permutation_polys, at --cpu-sizes only (2^20 and 2^22 by default); no extrapolation;
  * peak device memory of the call: the largest drop in free device memory, sampled by a second thread while the call
    runs, beside the library's own count (176 n bytes before the sort's temporary storage);
  * the GPU's S1..S3 are checked against permutation_polys wherever that ran.
With --profile, one more call at the largest size runs under torch.profiler (CUDA activities) for its kernel and copy
times.  The card's name and power limit are read in the same run.  Prints one JSON object; --out also writes it.

    python tools/permutation_bench.py --out profiles/h100_permutation.json --profile
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

MIB = 2 ** 20


class FreeMemorySampler:
    """lowest free device memory seen while the block runs (the library call releases the GIL)"""

    def __enter__(self):
        torch.cuda.synchronize()
        self.before = torch.cuda.mem_get_info()[0]
        self.low = self.before
        self.stop = False
        self.t = threading.Thread(target=self._run)
        self.t.start()
        return self

    def _run(self):
        while not self.stop:
            self.low = min(self.low, torch.cuda.mem_get_info()[0])
            time.sleep(0.0005)

    def __exit__(self, *exc):
        self.stop = True
        self.t.join()
        self.peak_bytes = self.before - self.low


def gpu_call(c, stream):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record(stream)
    S = pb.permutation_arrays(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
    end.record(stream)
    end.synchronize()
    return S, start.elapsed_time(end)


def profile_call(c):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        pb.permutation_arrays(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
        torch.cuda.synchronize()
    rows = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", 0) or 0
        if t > 0:
            rows[e.key[:120]] = round(t / 1e3, 3)
    return dict(sorted(rows.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--cpu-sizes", default="20,22", help="sizes at which permutation_polys runs once on the CPU")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--profile", action="store_true", help="one more call at the largest size under torch.profiler")
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this measures the GPU permutation")
    ctx = pb.default_context()
    stream = torch.cuda.ExternalStream(ctx.stream)
    res = {"device": torch.cuda.get_device_name(0)}
    try:
        res["power_limit_W"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        res["power_limit_W"] = None
    cpu_sizes = {int(x) for x in a.cpu_sizes.split(",") if x}
    res["sizes"] = []
    last = None
    for lg in (int(x) for x in a.sizes.split(",")):
        t = time.perf_counter()
        c = syn.build_circuit(lg, seed=7, n_public=2)
        r = {"log_n": lg, "circuit_build_s": round(time.perf_counter() - t, 1)}
        n = c.group_order
        S, r["warmup_ms"] = gpu_call(c, stream)
        ms = []
        with FreeMemorySampler() as mem:
            for _ in range(a.reps):
                S, t_ms = gpu_call(c, stream)
                ms.append(round(t_ms, 2))
        r["gpu_ms"] = ms
        r["gpu_ms_median"] = round(statistics.median(ms), 2)
        r["peak_device_MiB_sampled"] = round(mem.peak_bytes / MIB, 1)
        r["device_MiB_counted"] = round(176 * n / MIB, 1)
        if lg in cpu_sizes:
            t = time.perf_counter()
            want = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
            r["cpu_s"] = round(time.perf_counter() - t, 2)
            r["cpu_over_gpu"] = round(r["cpu_s"] * 1e3 / r["gpu_ms_median"], 1)
            for k in range(3):
                raw = b"".join(int(x).to_bytes(32, "little") for x in want[k])
                assert np.frombuffer(raw, dtype=np.uint8).reshape(-1, 32).tobytes() == S["S%d" % (k + 1)].tobytes(), k
            r["matches_cpu"] = True
            del want
        res["sizes"].append(r)
        print(json.dumps(r), flush=True)
        last = c
    if a.profile and last is not None:
        res["profile_log_n"] = last.group_order.bit_length() - 1
        try:
            res["profile_device_ms"] = profile_call(last)
        except Exception as e:  # the measurement above stands without the breakdown
            res["profile_error"] = repr(e)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(res, indent=1) + "\n")


if __name__ == "__main__":
    main()
