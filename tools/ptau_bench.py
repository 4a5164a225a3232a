"""Loading a ceremony SRS from a .ptau (Setup.from_ptau -> pb200_srs_create_ptau), split into its stages, against the
reference-shaped Setup.from_file.

Files are written first (sections 1, 2, 3 for the test tau, as tests/test_ptau.py writes them; the points come from
Setup.generate), for 2^k + 9 points at each --sizes k.  Each load is then timed as:
  * file read: np.fromfile of the tauG1 bytes (the page cache is warm: the file was just written; dropping it needs
    privileges a shared machine does not give);
  * pb200_srs_create_ptau on those bytes, host wall clock, and its stages (pb200_srs_ptau_stages): host-to-device copy
    through pinned staging, the check kernel k_ptau_check_g1 (CUDA events; 64 B per point over kernel time against the
    3.35 TB/s of the H100 SXM data sheet), the window table, the random scalars (getrandom), the consistency MSM
    (two vectors, one pass) and the pairing product, the [tau]_2 twist and subgroup checks;
  * Setup.from_ptau end to end (np.memmap of the same file).
One warm-up load per size first; the numbers are the median of --reps loads.  Setup.from_file is timed at --from-file
sizes on files whose power is that size (it reads 2^p points).  The card's name and power limit are read in the same
run.  Prints one JSON object; --out also writes it.

    python tools/ptau_bench.py --out profiles/h100_ptau.json
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
from concurrent.futures import ProcessPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import plonkathon_b200 as pb  # noqa: E402
from plonkathon_b200 import _lib  # noqa: E402
from plonkathon_b200.setup import ptau_layout  # noqa: E402

Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
HBM_BYTES_PER_S = 3.35e12
STAGES = ("h2d", "check_kernel", "window_table", "random_scalars", "consistency_msm", "pairing", "tau_g2_checks")
G2_GEN = (10857046999023057135944570762232829481370756359578518086990519993285655852781,
          11559732032986387107991004021392285783925812861821192530917403151452391805634,
          8495653923123431417604973247489272438418190587263600148770280649306958101930,
          4082367875863433681332203403145435568316851327593401208105741076214120093531)


def to_mont(raw: bytes) -> bytes:
    rm = pow(2, 256, Q)
    return b"".join((int.from_bytes(raw[i:i + 32], "little") * rm % Q).to_bytes(32, "little")
                    for i in range(0, len(raw), 32))


def write_ptau(path, power, count, pool):
    gen = pb.Setup.generate(TAU, count, precompute=False)
    step = 1 << 18
    x2 = gen.X2
    tau_g2 = to_mont(b"".join(c.n.to_bytes(32, "little") for coord in x2 for c in coord.coeffs))
    header = (32).to_bytes(4, "little") + Q.to_bytes(32, "little") + power.to_bytes(4, "little") * 2
    g2 = to_mont(b"".join(c.to_bytes(32, "little") for c in G2_GEN)) + tau_g2
    with open(path, "wb") as f:
        f.write(b"ptau" + (1).to_bytes(4, "little") + (3).to_bytes(4, "little"))
        f.write((1).to_bytes(4, "little") + len(header).to_bytes(8, "little") + header)
        f.write((2).to_bytes(4, "little") + (64 * count).to_bytes(8, "little"))
        parts = [gen.export_points_array(i, min(step, count - i)).tobytes() for i in range(0, count, step)]
        for chunk in pool.map(to_mont, parts):
            f.write(chunk)
        f.write((3).to_bytes(4, "little") + len(g2).to_bytes(8, "little") + g2)
    del gen


def load_once(path):
    with open(path, "rb") as f:
        sec = ptau_layout(f)
        g1_off, g1_size, _ = sec[2]
        f.seek(sec[3][0] + 128)
        tau_g2 = f.read(128)
    count = g1_size // 64
    t0 = time.perf_counter()
    g1 = np.fromfile(path, dtype=np.uint8, count=g1_size, offset=g1_off)
    t_read = time.perf_counter() - t0
    ctx = pb.default_context()
    h = ctypes.c_void_p()
    t0 = time.perf_counter()
    _lib.check(_lib.lib().pb200_srs_create_ptau(ctx.handle, g1.ctypes.data_as(ctypes.c_void_p), count, tau_g2, 1,
                                                ctypes.byref(h)))
    t_lib = time.perf_counter() - t0
    ms = (ctypes.c_double * len(STAGES))()
    _lib.lib().pb200_srs_ptau_stages(ms, len(STAGES))
    _lib.lib().pb200_srs_destroy(h)
    del g1
    t0 = time.perf_counter()
    s = pb.Setup.from_ptau(path, powers=count)
    t_e2e = time.perf_counter() - t0
    del s
    return {"file_read_ms": 1e3 * t_read, "library_load_ms": 1e3 * t_lib,
            "from_ptau_end_to_end_ms": 1e3 * t_e2e, **{k + "_ms": ms[i] for i, k in enumerate(STAGES)}}


def median_of(runs):
    return {k: statistics.median(r[k] for r in runs) for k in runs[0]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="20,22,24")
    ap.add_argument("--from-file", default="16,20")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()[0]
    res = {"gpu": smi, "page_cache": "warm (files read right after they were written)", "loads": {}, "from_file": {}}
    tmp = tempfile.mkdtemp(prefix="pb200_ptau_")
    with ProcessPoolExecutor(max_workers=min(32, os.cpu_count() or 1)) as pool:
        for k in [int(x) for x in a.sizes.split(",") if x]:
            count = (1 << k) + 9
            path = os.path.join(tmp, "p%d.ptau" % k)
            t0 = time.perf_counter()
            write_ptau(path, k, count, pool)
            write_s = time.perf_counter() - t0
            load_once(path)  # warm-up: module load, pairing constants, pinned allocations
            m = median_of([load_once(path) for _ in range(a.reps)])
            m["check_kernel_GBps"] = 64 * count / (m["check_kernel_ms"] * 1e-3) / 1e9
            m["check_kernel_share_of_3.35TBps"] = 64 * count / (m["check_kernel_ms"] * 1e-3) / HBM_BYTES_PER_S
            m["check_share_of_library_load"] = m["check_kernel_ms"] / m["library_load_ms"]
            res["loads"]["2^%d+9" % k] = {"points": count, "file_bytes": os.path.getsize(path),
                                          "write_file_s": write_s, **m}
            os.remove(path)
            print(json.dumps({k: res["loads"]["2^%d+9" % k]}), file=sys.stderr, flush=True)
        for k in [int(x) for x in a.from_file.split(",") if x]:
            path = os.path.join(tmp, "f%d.ptau" % k)
            write_ptau(path, k, 1 << k, pool)
            t0 = time.perf_counter()
            s = pb.Setup.from_file(path)
            t_ff = time.perf_counter() - t0
            del s
            t0 = time.perf_counter()
            s = pb.Setup.from_ptau(path)
            t_fp = time.perf_counter() - t0
            del s
            res["from_file"]["2^%d" % k] = {"from_file_ms": 1e3 * t_ff, "from_ptau_ms": 1e3 * t_fp}
            os.remove(path)
    res["from_file"]["2^24"] = "not measured"
    out = json.dumps(res, indent=1)
    print(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(out + "\n")


if __name__ == "__main__":
    main()
