"""Time solve_wires with a table argument (csrc/solve.cu, pb200_solve_wires_lookup) on table circuits.

table: synthetic.table_circuit, tagged (range, XOR and AND tables, 4-bit operands), solved from its seeds:
       deep  one chain: every row depends on the row before it;
       wide  2^16 chains interleaved (fewer where 2^16 six-row steps do not fit: n / 16 chains).
step:  one chain of n rows where every row reads the two before it, all gate rows (c = a + b) or all table rows
       (c = a ^ b from a 4-bit XOR table): the cost of one dependent table step against one dependent gate step.

Per run: the rows, the defining rows, the depth (longest chain of defining rows, on the host), the device time of the
library call (CUDA events on the context's stream around it), the end-to-end time of solve_wires from host arrays to
device tensors, and the device time per dependent step.  At 2^20 the tagged deep circuit is also solved by a Python
restatement of the rule and the two results compared.  The card's name and power limit are read in the same run.
Prints one JSON line per run; --out also writes the whole series to a file, after every run.

    python tools/solve_lookup_bench.py [--sizes 16,20,22] --out profiles/h100_solve_lookup.json
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
from plonkathon_b200.lookup import check_lookups, xor_table  # noqa: E402

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


def table(log_n, chains):
    c = syn.table_circuit(log_n, chains=chains, seed=log_n)
    ins = {v: c.values[v] for v in range(2 * chains)}
    return c, ins, {"lookups": syn.lookups_arrays(c)}


def step_chain(log_n, kind):
    """n rows, row r: v(r + 2) = v(r) op v(r + 1); op = a + b (gate) or a ^ b (one XOR table of 4 bits)"""
    n = 1 << log_n
    r = np.arange(n, dtype=np.int64)
    sel = {k: [0] * n for k in SEL}
    if kind == "gate":
        sel["QL"] = sel["QR"] = [R - 1] * n
        sel["QO"] = [1] * n
        kw, qk = {}, None
    else:
        qk = [1] * n
        kw = {"lookup": (qk, xor_table(4))}
    c = syn.ArrayCircuit(n, n, r, r + 1, r + 2, sel["QL"], sel["QR"], sel["QM"], sel["QO"], sel["QC"], 0, [], [])
    return c, {0: 3, 1: 5}, kw


def depth_of(c, ins, kw):
    """the longest chain of defining rows under the rule, on the host"""
    m = c.n_constraints
    qk = check_lookups(kw["lookups"], c.group_order)[0] if "lookups" in kw else (kw["lookup"][0] if kw else None)
    depth, best = {v: 0 for v in ins}, 0
    depth[-1] = 0
    L, Rw, O = (np.asarray(w[:m]).tolist() for w in (c.wire_L, c.wire_R, c.wire_O))
    for r in range(m):
        v = O[r]
        if v < 0 or v in depth:
            continue
        if c.QO[r] != 0 or (qk is not None and qk[r]):
            depth[v] = d = 1 + max(depth[L[r]], depth[Rw[r]])
            best = max(best, d)
    return best


def restate(c, ins, kw):
    """the C column by the Python restatement of the rule (tests/test_solve_lookup.py restates it in full)"""
    qk, qt, cols, _ = check_lookups(kw["lookups"], c.group_order)
    index = {(cols[3][i], cols[0][i], cols[1][i]): cols[2][i] for i in range(len(cols[0]))}
    val = {-1: 0}
    val.update(ins)
    m = c.n_constraints
    L, Rw, O = (np.asarray(w[:m]).tolist() for w in (c.wire_L, c.wire_R, c.wire_O))
    for r in range(m):
        v = O[r]
        if v < 0 or v in val:
            continue
        a, b = val[L[r]], val[Rw[r]]
        if c.QO[r] == 0 and qk[r]:
            val[v] = index[(qt[r], a, b)]
        elif c.QO[r] != 0:
            s = c.QL[r] * a + c.QR[r] * b + c.QM[r] * a * b + c.QC[r]
            val[v] = -s * pow(c.QO[r], R - 2, R) % R
    return [val[v] for v in O]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="16,20,22")
    ap.add_argument("--step-sizes", default="16,20")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    args = ap.parse_args()
    import torch
    stream = torch.cuda.Stream()
    ctx = pb.Context(0, stream=stream.cuda_stream)
    res = {"card": card(), "runs": []}
    print(res["card"], flush=True)
    cases = []
    for log_n in [int(x) for x in args.sizes.split(",") if x]:
        cases.append((log_n, "table_deep", lambda ln=log_n: table(ln, 1)))
        cases.append((log_n, "table_wide", lambda ln=log_n: table(ln, min(WIDE, (1 << ln) // 16))))
    for log_n in [int(x) for x in args.step_sizes.split(",") if x]:
        cases.append((log_n, "step_gate", lambda ln=log_n: step_chain(ln, "gate")))
        cases.append((log_n, "step_table", lambda ln=log_n: step_chain(ln, "table")))
    for log_n, name, make in cases:
        t0 = time.time()
        c, ins, kw = make()
        n = c.group_order
        pk = {k: le(getattr(c, k)) for k in SEL}
        in_ids = np.array(list(ins), np.int64)
        in_vals = le(list(ins.values()))
        depth = depth_of(c, ins, kw)
        run = {"log_n": log_n, "circuit": name, "rows": c.n_constraints, "inputs": len(ins), "depth": depth,
               "host_build_s": round(time.time() - t0, 1)}

        def solve():
            return pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, pk, (in_ids, in_vals), n,
                                  n_constraints=c.n_constraints, device=True, ctx=ctx, **kw)
        sol = solve()  # warm-up
        assert sol.ok, str(sol)
        dev, e2e = [], []
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
            e2e.append((time.perf_counter() - t1) * 1e3)
            dev.append(a.elapsed_time(b))
        run["solve_device_ms"] = round(min(dev), 2)
        run["solve_e2e_ms"] = round(min(e2e), 2)
        run["ns_per_dependent_step"] = round(min(dev) * 1e6 / depth, 1)
        if name == "table_deep":
            want = c.wires_values()[2]
            assert np.array_equal(sol.C.cpu().numpy(), le(want)), "solve_wires disagrees with wires_values()"
            run["equals_wires_values"] = True
        if log_n == 20 and name == "table_deep":
            t1 = time.perf_counter()
            col = restate(c, ins, kw)
            run["python_restatement_ms"] = round((time.perf_counter() - t1) * 1e3, 1)
            assert col == list(want[:c.n_constraints]), "the restatement disagrees with wires_values()"
        del sol
        print(json.dumps(run), flush=True)
        res["runs"].append(run)
        if args.out:
            os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
            with open(args.out, "w") as f:  # after every run, so a partial series is kept
                json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
