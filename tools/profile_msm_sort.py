"""Kernel times of tools/one_commit.py (fixed-base commitments of 2^k random coefficients, the prover's MSM
shape) under torch.profiler with CUDA activities: one row per kernel name, summed over the timed commitments.

    python tools/profile_msm_sort.py [log_n] [out.md]

The first commitment warms up (module load, scratch allocation) and is not profiled; the next three are."""
import ctypes, os, sys, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import profile, ProfilerActivity
import plonkathon_b200 as pb
from plonkathon_b200 import _lib

logn = int(sys.argv[1]) if len(sys.argv) > 1 else 20
out_md = sys.argv[2] if len(sys.argv) > 2 else None
REPS = 3
L = _lib.lib(); ctx = _lib.default_context()
n = 1 << logn
setup = pb.Setup.generate(0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF, n, ctx=ctx)
x = torch.randint(0, 2 ** 31 - 1, (n, 8), dtype=torch.int32, device="cuda"); x[:, 7] &= 0x0FFFFFFF
out = ctypes.create_string_buffer(64); ident = ctypes.c_int()


def commit():
    _lib.check(L.pb200_srs_commit_coeffs(ctx.handle, setup._srs, ctypes.c_void_p(x.data_ptr()), n, 0, out, ctypes.byref(ident)))


commit()
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(REPS):
        commit()
    torch.cuda.synchronize()

rows = {}
for ev in prof.events():
    if ev.device_type != torch.autograd.DeviceType.CUDA:
        continue
    name = ev.name.split("(")[0].split("<")[0].replace("pb200::", "").strip()
    r = rows.setdefault(name, [0, 0.0])
    r[0] += 1
    r[1] += ev.device_time / 1e3
gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                     text=True).stdout.strip()
lines = [f"GPU: {gpu}", f"{REPS} fixed-base commitments of 2^{logn} coefficients (batch 1), per commitment:", "",
         "| kernel | launches | ms |", "|---|---|---|"]
total = 0.0
for name, (cnt, ms) in sorted(rows.items(), key=lambda kv: -kv[1][1]):
    lines.append(f"| {name} | {cnt // REPS} | {ms / REPS:.3f} |")
    total += ms / REPS
lines.append(f"| total | | {total:.3f} |")
text = "\n".join(lines)
print(text)
if out_md:
    os.makedirs(os.path.dirname(os.path.abspath(out_md)), exist_ok=True)
    with open(out_md, "w") as f:
        f.write(text + "\n")
