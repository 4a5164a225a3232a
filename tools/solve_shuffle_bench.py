"""Time solve_wires with a shuffle (csrc/solve.cu, pb200_solve_wires_shuffle).

memory: synthetic.memory_circuit (2^(log_n - 6) addresses), solved from its seeds: the library call's device time
        (CUDA events on the context's stream around it), split into phase 1 (the defining rows below the first
        out-row), the shuffle step and phase 2 (pb200_solve_shuffle_stages, device events inside the call), and the
        end-to-end time of solve_wires from host arrays to device tensors.  The wires are compared with the builder's.
sort:   the shuffle step alone: K = n/4 in-rows whose cells are inputs and K out-rows after them, no gates.
        small:  (address < 2^10, time = the record's index, value < 2^16): one or two sort passes a word;
        random: three random field elements: all twelve words sorted.
At 2^20 the memory circuit is also solved by the Python restatement (tests/test_solve_shuffle.py) and the two results
compared.  The card's name and power limit are read in the same run.  Prints one JSON line per run; --out writes the
whole series, --md a table of it, after every run.

    python tools/solve_shuffle_bench.py [--sizes 20,22] --out profiles/h100_solve_shuffle.json \
        --md profiles/h100_solve_shuffle_ab.md
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import _lib  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402

R = syn.R
SEL = ("QL", "QR", "QM", "QO", "QC")


def le(ints):
    """ints -> (n, 32) uint8, through four 64-bit words (no per-value bytes objects)"""
    a = np.array([int(x) for x in ints], dtype=object)
    out = np.empty((len(a), 4), np.uint64)
    for w in range(4):
        out[:, w] = ((a >> (64 * w)) & (2**64 - 1)).astype(np.uint64)
    return out.view(np.uint8).reshape(-1, 32)


def memory(log_n):
    n_addr = 1 << (log_n - 6)
    c = syn.memory_circuit(log_n, n_addr, seed=log_n)
    ins = list(range(2 * n_addr + 2))
    pk = {k: le(getattr(c, k)) for k in SEL}
    return c, pk, (np.array(ins, np.int64), le([c.values[v] for v in ins]))


def sort_only(log_n, kind, seed=1):
    """K = n/4 input records on rows [0, K), K out-rows of fresh variables on rows [K, 2K)"""
    n = 1 << log_n
    K = n // 4
    rng = np.random.default_rng(seed)
    words = np.zeros((3 * K, 4), np.uint64)
    if kind == "small":
        words[0::3, 0] = rng.integers(0, 1 << 10, K, dtype=np.uint64)
        words[1::3, 0] = np.arange(K, dtype=np.uint64)
        words[2::3, 0] = rng.integers(0, 1 << 16, K, dtype=np.uint64)
    else:
        words[:, :3] = rng.integers(0, 2**64, (3 * K, 3), dtype=np.uint64, endpoint=False)
        words[:, 3] = rng.integers(0, 0x3064 << 48, 3 * K, dtype=np.uint64)  # below r
    ids = np.full((n, 3), -1, np.int64)
    ids[:2 * K] = np.arange(6 * K, dtype=np.int64).reshape(2 * K, 3)
    q = np.zeros(n, np.int64)
    q_in, q_out = q.copy(), q.copy()
    q_in[:K] = 1
    q_out[K:2 * K] = 1
    c = syn.ArrayCircuit(n, 2 * K, ids[:, 0], ids[:, 1], ids[:, 2], *([[0] * n] * 5), 0, [], [],
                         shuffle=(q_in.tolist(), q_out.tolist()))
    pk = {k: np.zeros((n, 32), np.uint8) for k in SEL}
    return c, pk, (np.arange(3 * K, dtype=np.int64), words.view(np.uint8).reshape(-1, 32))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def write_md(path, res):
    rows = ["| log_n | circuit | in-rows | solve (device) ms | phase 1 ms | shuffle ms | phase 2 ms | e2e ms |",
            "|---|---|---|---|---|---|---|---|"]
    for r in res["runs"]:
        rows.append("| %d | %s | %d | %.2f | %.2f | %.2f | %.2f | %.2f |" % (
            r["log_n"], r["circuit"], r["in_rows"], r["solve_device_ms"], r["phase1_ms"], r["shuffle_ms"],
            r["phase2_ms"], r["solve_e2e_ms"]))
    py = [r for r in res["runs"] if "python_restatement_ms" in r]
    text = ["# solve_wires with a shuffle", "", "Card: %s (name, power limit, max SM clock, read in the same run)."
            % res["card"], "", "Best of %d calls after a warm-up (tools/solve_shuffle_bench.py)." % res["reps"], ""]
    text += rows
    if py:
        text += ["", "Python restatement of the rule at 2^%d: %.1f s, equal to the library's wires."
                 % (py[0]["log_n"], py[0]["python_restatement_ms"] / 1e3)]
    with open(path, "w") as f:
        f.write("\n".join(text) + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out")
    ap.add_argument("--md")
    args = ap.parse_args()
    import torch
    stream = torch.cuda.Stream()
    ctx = pb.Context(0, stream=stream.cuda_stream)
    res = {"card": card(), "reps": args.reps, "runs": []}
    print(res["card"], flush=True)
    cases = []
    for log_n in [int(x) for x in args.sizes.split(",") if x]:
        cases.append((log_n, "memory", lambda ln=log_n: memory(ln)))
        cases.append((log_n, "sort_small", lambda ln=log_n: sort_only(ln, "small")))
        cases.append((log_n, "sort_random", lambda ln=log_n: sort_only(ln, "random")))
    stages = (ctypes.c_double * 3)()
    for log_n, name, make in cases:
        t0 = time.time()
        c, pk, ins = make()
        n = c.group_order
        run = {"log_n": log_n, "circuit": name, "rows": c.n_constraints, "in_rows": int(sum(c.shuffle[0])),
               "host_build_s": round(time.time() - t0, 1)}
        cust = syn.custom_arrays(c)

        def solve():
            return pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, pk, ins, n, n_constraints=c.n_constraints,
                                  custom=cust, shuffle=c.shuffle, device=True, ctx=ctx)
        sol = solve()  # warm-up
        assert sol.ok, str(sol)
        best = None
        for _ in range(args.reps):
            del sol
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t1 = time.perf_counter()
            with torch.cuda.stream(stream):
                a.record(stream)
                sol = solve()
                b.record(stream)
            b.synchronize()
            e2e = (time.perf_counter() - t1) * 1e3
            _lib.lib().pb200_solve_shuffle_stages(stages, 3)
            got = (a.elapsed_time(b), list(stages), e2e)
            if best is None or got[0] < best[0]:
                best = got
        run["solve_device_ms"] = round(best[0], 2)
        run["phase1_ms"], run["shuffle_ms"], run["phase2_ms"] = (round(x, 2) for x in best[1])
        run["solve_e2e_ms"] = round(best[2], 2)
        C = sol.C.cpu().numpy()
        if name == "memory":
            want = c.wires_values()
            assert np.array_equal(C, le(want[2])), "solve_wires disagrees with wires_values()"
            run["equals_wires_values"] = True
        else:
            K = run["in_rows"]
            tup = np.stack([X.cpu().numpy()[K:2 * K] for X in (sol.A, sol.B, sol.C)], axis=1).reshape(K, 96)
            rec = ins[1].reshape(K, 96)
            key = lambda t: [bytes(x[::-1]) for x in t.reshape(3, 32)]  # noqa: E731
            assert sorted(key(t) for t in rec) == [key(t) for t in tup], "the out-rows are not the sorted in-rows"
            run["equals_sorted"] = True
        if log_n == 20 and name == "memory":
            sys.path.insert(0, ROOT)
            from tests.test_solve_shuffle import _restate, memory_seeds
            t1 = time.perf_counter()
            cols = _restate(c, memory_seeds(c, 1 << (log_n - 6)))[0]
            run["python_restatement_ms"] = round((time.perf_counter() - t1) * 1e3, 1)
            assert cols[2] == list(want[2]), "the restatement disagrees with wires_values()"
        del sol
        print(json.dumps(run), flush=True)
        res["runs"].append(run)
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            with open(args.out, "w") as f:  # after every run, so a partial series is kept
                json.dump(res, f, indent=1)
        if args.md:
            write_md(args.md, res)


if __name__ == "__main__":
    main()
