"""Where the proofs in flight overlap: K prover lanes (own context and stream, shared SRS, one host thread each, as
bench.py runs them) prove a few 2^20-gate proofs under torch.profiler with CUDA activities.  Every kernel is given to
the lane whose host thread launched it (runtime-API correlation ids; lanes are numbered in the order of their
threads' ids in the trace) and to a phase by its name.  For each lane and
phase the tool prints the kernel time, the share of it during which a kernel of another lane runs (any kernel, and
an MSM bucket accumulation), and the lane's idle time in front of the phase's kernels.

Usage: python tools/inflight_trace.py [--lanes K] [--proofs P] [--warmup W] [--out DIR]
The Chrome trace and the table (JSON) go to DIR (a temporary directory by default)."""
import argparse
import bisect
import ctypes
import json
import os
import re
import sys
import tempfile
from collections import Counter
from concurrent.futures import ThreadPoolExecutor

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PHASES = ("sort", "accumulate", "stitch", "reduce0", "reduce_upper", "ntt", "quotient", "other")


def phase_of(kernel):
    if kernel.startswith(("k_msm_bin_", "k_msm_chunk_", "k_scan_")):
        return "sort"
    if kernel == "k_msm_seg_accumulate":
        return "accumulate"
    if kernel.startswith("k_msm_stitch"):
        return "stitch"
    if kernel == "k_reduce_level0":
        return "reduce0"
    if kernel == "k_reduce_block":
        return "reduce_upper"
    if kernel.startswith("k_ntt"):
        return "ntt"
    if kernel.startswith("k_quotient"):
        return "quotient"
    return "other"


def merge(iv):
    """union of [a, b) intervals, sorted and disjoint"""
    out = []
    for a, b in sorted(iv):
        if out and a <= out[-1][1]:
            out[-1][1] = max(out[-1][1], b)
        else:
            out.append([a, b])
    return out


def covered(a, b, merged, starts):
    """length of [a, b) that lies inside the union `merged` (starts: its left ends, for bisection)"""
    i = max(0, bisect.bisect_right(starts, a) - 1)
    s = 0.0
    while i < len(merged) and merged[i][0] < b:
        s += max(0.0, min(b, merged[i][1]) - max(a, merged[i][0]))
        i += 1
    return s


def kernels_by_lane(trace, lanes):
    """[(lane, kernel name, start us, end us)] from a Chrome trace of torch.profiler: the `lanes` host threads that
    launched the most kernels are the lanes"""
    corr_tid = {}
    for e in trace["traceEvents"]:
        if e.get("cat") in ("cuda_runtime", "cuda_driver") and "correlation" in e.get("args", {}):
            corr_tid[e["args"]["correlation"]] = e["tid"]
    launches = Counter(corr_tid.get(e["args"].get("correlation")) for e in trace["traceEvents"] if e.get("cat") == "kernel")
    launches.pop(None, None)
    thread_lane = {tid: k for k, tid in enumerate(sorted(t for t, _ in launches.most_common(lanes)))}
    out = []
    for e in trace["traceEvents"]:
        if e.get("cat") != "kernel":
            continue
        tid = corr_tid.get(e["args"].get("correlation"))
        if tid not in thread_lane:
            continue
        m = re.search(r"\b(k_[A-Za-z0-9_]+)", e["name"])
        name = m.group(1) if m else e["name"]
        out.append((thread_lane[tid], name, float(e["ts"]), float(e["ts"]) + float(e["dur"])))
    return out


def analyse(kernels, lanes):
    res = {}
    t0 = min(k[2] for k in kernels)
    t1 = max(k[3] for k in kernels)
    for lane in range(lanes):
        mine = sorted((k for k in kernels if k[0] == lane), key=lambda k: k[2])
        others = merge([[k[2], k[3]] for k in kernels if k[0] != lane])
        others_acc = merge([[k[2], k[3]] for k in kernels if k[0] != lane and k[1] == "k_msm_seg_accumulate"])
        os_, oas = [m[0] for m in others], [m[0] for m in others_acc]
        ph = {p: {"kernels": 0, "ms": 0.0, "with_other_ms": 0.0, "with_other_acc_ms": 0.0, "idle_before_ms": 0.0}
              for p in PHASES}
        busy_end = t0
        for _, name, a, b in mine:
            d = ph[phase_of(name)]
            d["kernels"] += 1
            d["ms"] += (b - a) / 1e3
            d["with_other_ms"] += covered(a, b, others, os_) / 1e3
            d["with_other_acc_ms"] += covered(a, b, others_acc, oas) / 1e3
            d["idle_before_ms"] += max(0.0, a - busy_end) / 1e3
            busy_end = max(busy_end, b)
        busy = sum(b - a for a, b in merge([[k[2], k[3]] for k in mine]))
        res[lane] = {"phases": ph, "window_ms": (t1 - t0) / 1e3, "busy_ms": busy / 1e3,
                     "idle_ms": (t1 - t0 - busy) / 1e3}
    return res


def print_table(res, proofs):
    print("| lane | phase | kernels | ms per proof | with another lane's kernel | with another lane's accumulation | "
          "lane idle before it, ms per proof |")
    print("|---|---|---|---|---|---|---|")
    for lane, r in res.items():
        for p in PHASES:
            d = r["phases"][p]
            if not d["kernels"]:
                continue
            f = d["with_other_ms"] / d["ms"] if d["ms"] else 0.0
            fa = d["with_other_acc_ms"] / d["ms"] if d["ms"] else 0.0
            print("| %d | %s | %d | %.2f | %.0f %% | %.0f %% | %.2f |"
                  % (lane, p, d["kernels"] // proofs, d["ms"] / proofs, 100 * f, 100 * fa, d["idle_before_ms"] / proofs))
    for lane, r in res.items():
        print("lane %d: window %.1f ms, kernels running %.1f ms, idle %.1f ms (%.2f ms per proof)"
              % (lane, r["window_ms"], r["busy_ms"], r["idle_ms"], r["idle_ms"] / proofs))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=2)
    ap.add_argument("--proofs", type=int, default=3, help="traced proofs per lane")
    ap.add_argument("--warmup", type=int, default=2, help="untraced proofs per lane first")
    ap.add_argument("--log-n", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import numpy as np
    import torch
    from torch.profiler import ProfilerActivity, profile
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, synthetic as syn

    out = args.out or tempfile.mkdtemp(prefix="inflight_trace_")
    os.makedirs(out, exist_ok=True)
    L = _lib.lib()
    n = 1 << args.log_n
    ctx0 = _lib.Context(0)
    setup = pb.Setup.generate(0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF, n, ctx=ctx0)
    circ = syn.build_circuit(args.log_n, seed=20260924, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(circ)
    pub = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in public), dtype=np.uint8).reshape(-1, 32).copy()
    vp = ctypes.c_void_p
    lanes = []
    for k in range(args.lanes):
        ctx = ctx0 if k == 0 else _lib.Context(0)
        d = tuple(torch.from_numpy(x.copy()).cuda() for x in (A, B, C))
        lanes.append(dict(prover=pb.Prover.from_arrays(setup, n, pk, ctx=ctx), d=d, proof=ctypes.create_string_buffer(768)))

    def prove(lane):
        _lib.check(L.pb200_prover_prove_device(lane["prover"]._h, *[vp(t.data_ptr()) for t in lane["d"]],
                                               pub.ctypes.data_as(vp), pub.shape[0], lane["proof"]))

    def worker(k, steps):
        for _ in range(steps):
            prove(lanes[k])

    pool = ThreadPoolExecutor(args.lanes)
    list(pool.map(lambda k: worker(k, args.warmup), range(args.lanes)))
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        list(pool.map(lambda k: worker(k, args.proofs), range(args.lanes)))
        torch.cuda.synchronize()
    pool.shutdown()
    ref = lanes[0]["proof"].raw
    assert all(l["proof"].raw == ref for l in lanes), "lanes disagree"
    path = os.path.join(out, "inflight.pt.trace.json")
    prof.export_chrome_trace(path)
    with open(path) as f:
        trace = json.load(f)
    kernels = kernels_by_lane(trace, args.lanes)
    res = analyse(kernels, args.lanes)
    dev = torch.cuda.get_device_properties(0)
    print("device: %s; %d lanes x %d traced proofs of 2^%d gates" % (dev.name, args.lanes, args.proofs, args.log_n))
    print_table(res, args.proofs)
    with open(os.path.join(out, "inflight_trace.json"), "w") as f:
        json.dump({"device": dev.name, "lanes": args.lanes, "proofs": args.proofs, "log_n": args.log_n,
                   "result": {str(k): v for k, v in res.items()}}, f, indent=1)
    print("trace and table:", out)


if __name__ == "__main__":
    main()
