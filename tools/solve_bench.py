"""Time solve_wires (csrc/solve.cu) on a deep and a wide circuit at 2^20, 2^22 and 2^24 rows.

deep: the synthetic bench circuit (synthetic.build_circuit, seed 7): each gate's operands come from the 64 most
      recently produced variables, so the chain of defining rows is long.
wide: 2^16 independent chains of a + b / a * b rows, interleaved, built with numpy: depth n / 2^16.

Per size and circuit: the depth (longest chain of defining rows, on the host), the device time of the library call
(CUDA events on the context's stream around it: the sort, the checks, the evaluation and the writes, with the call's
host round trips inside), the end-to-end time of solve_wires from host arrays to device tensors, and at 2^20 the
time of a Python restatement of the rule.  The card's name and power limit are read in the same run.  Prints one JSON
line per run; --out also writes the whole series to a file, after every run.

    python tools/solve_bench.py [--sizes 20,22,24] --out profiles/h100_solve.json
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

R = syn.R
SEL = ("QL", "QR", "QM", "QO", "QC")
WIDE = 1 << 16


def le(ints):
    """ints -> (n, 32) uint8, through four 64-bit words (no per-value bytes objects)"""
    a = np.array([int(x) for x in ints], dtype=object)
    out = np.empty((len(a), 4), np.uint64)
    for w in range(4):
        out[:, w] = ((a >> (64 * w)) & (2**64 - 1)).astype(np.uint64)
    return out.view(np.uint8).reshape(-1, 32)


def deep(log_n):
    c = syn.build_circuit(log_n, seed=7, n_public=2)
    return c.wire_L, c.wire_R, c.wire_O, {k: getattr(c, k) for k in SEL}, c.n_constraints, c.values


def wide(log_n):
    n = 1 << log_n
    rng = np.random.default_rng(1)
    r = np.arange(n)
    k, step = r % WIDE, r // WIDE
    O = 2 * WIDE + r
    prev = np.where(step >= 1, O - WIDE, k)                # the chain's previous output, or its first input
    prev2 = np.where(step >= 2, O - 2 * WIDE, np.where(step == 1, k, WIDE + k))
    mul = rng.integers(0, 2, n).astype(bool)
    add = [0 if x else R - 1 for x in mul.tolist()]
    sel = {"QL": add, "QR": add, "QM": [R - 1 if x else 0 for x in mul.tolist()], "QO": [1] * n, "QC": [0] * n}
    values = [int(x) for x in rng.integers(1, 2**62, 2 * WIDE)]
    return prev, prev2, O, sel, n, values


def defining(L, Rw, O, sel, m):
    """row of each defined variable (first row with it on O and QO != 0), the inputs, the depth"""
    O = np.asarray(O[:m])
    qo = np.array([x != 0 for x in sel["QO"][:m]])
    rows = np.flatnonzero((O >= 0) & qo)
    vars_, first = np.unique(O[rows], return_index=True)
    def_row = dict(zip(vars_.tolist(), rows[first].tolist()))
    used = set(np.asarray(L[:m]).tolist()) | set(np.asarray(Rw[:m]).tolist()) | set(O.tolist())
    used.discard(-1)
    inputs = sorted(used - set(def_row))
    depth = {}
    best = 0
    for v, r in sorted(def_row.items(), key=lambda t: t[1]):
        d = 1 + max(depth.get(int(L[r]), 0), depth.get(int(Rw[r]), 0))
        depth[v] = d
        best = max(best, d)
    return def_row, inputs, best


def restate(L, Rw, O, sel, m, def_row, inputs, values):
    val = {-1: 0}
    val.update((v, values[v]) for v in inputs)
    for r in sorted(def_row.values()):
        a, b = val[int(L[r])], val[int(Rw[r])]
        s = sel["QL"][r] * a + sel["QR"][r] * b + sel["QM"][r] * a * b + sel["QC"][r]
        val[int(O[r])] = -s * pow(sel["QO"][r], R - 2, R) % R
    return val


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    stream = torch.cuda.Stream()
    ctx = pb.Context(0, stream=stream.cuda_stream)
    res = {"card": card(), "runs": []}
    print(res["card"], flush=True)
    for log_n in [int(x) for x in args.sizes.split(",")]:
        for name, make in (("deep", deep), ("wide", wide)):
            t0 = time.time()
            L, Rw, O, sel, m, values = make(log_n)
            n = 1 << log_n
            def_row, inputs, depth = defining(L, Rw, O, sel, m)
            pk = {k: le(sel[k]) for k in SEL}
            in_ids = np.array(inputs, np.int64)
            in_vals = le([values[v] for v in inputs])
            build_s = time.time() - t0
            run = {"log_n": log_n, "circuit": name, "rows": m, "defining_rows": len(def_row), "inputs": len(inputs),
                   "depth": depth, "host_build_s": round(build_s, 1)}
            sol = pb.solve_wires(L, Rw, O, pk, (in_ids, in_vals), n, n_constraints=m, device=True, ctx=ctx)  # warm-up
            assert sol.ok, str(sol)
            dev, e2e = [], []
            for _ in range(args.reps):
                del sol
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t1 = time.perf_counter()
                with torch.cuda.stream(stream):
                    a.record(stream)
                    sol = pb.solve_wires(L, Rw, O, pk, (in_ids, in_vals), n, n_constraints=m, device=True, ctx=ctx)
                    b.record(stream)
                b.synchronize()
                e2e.append((time.perf_counter() - t1) * 1e3)
                dev.append(a.elapsed_time(b))
            run["solve_device_ms"] = round(min(dev), 2)
            run["solve_e2e_ms"] = round(min(e2e), 2)
            run["ns_per_dependent_step"] = round(min(dev) * 1e6 / depth, 1)
            if log_n == 20:
                t1 = time.perf_counter()
                val = restate(L, Rw, O, sel, m, def_row, inputs, values)
                run["python_restatement_ms"] = round((time.perf_counter() - t1) * 1e3, 1)
                got = sol.C.cpu().numpy()
                want = le([val[int(v)] if v >= 0 else 0 for v in np.asarray(O[:m])])
                assert np.array_equal(got[:m], want), "solve_wires disagrees with the restatement"
                run["equals_restatement"] = True
            del sol
            print(json.dumps(run), flush=True)
            res["runs"].append(run)
            if args.out:
                os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
                with open(args.out, "w") as f:  # after every run, so a partial series is kept
                    json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
