"""Multi-GPU: one process per GPU (torchrun), ``torch.distributed`` for the plumbing.

Two modes:

* replicas (bench.py's headline at N > 1): proofs are independent units, every rank owns an SRS replica and
  proves its own instances -- no data-path collective.

* ONE proof across the GPUs of a box (north_star: "shard MSM ... and NTT by coefficient-slab ... with a single NCCL
  allgather at the join"): every rank holds the witness, the circuit and an SRS replica and runs the same
  ``Prover.prove``; inside the library (csrc/prover.cu, world > 1)
    - rank r owns every G-th point of the 4n coset, so the coset extensions, the cached selector extensions and the
      quotient are local and divide by G;
    - Lagrange -> coefficient transforms are slab-sharded: local n/G-point transforms, ONE allgather, a G-point DFT
      per element at the join (csrc/ntt_shard.cuh);
    - every commitment splits its 2^(c-1) buckets over the ranks (accumulation AND reduction divide by G), with ONE
      allgather of 256 bytes per rank at the join (csrc/msm.cu).
  The collectives are issued by the library itself on its CUDA stream through its own NCCL communicator
  (csrc/comm.cu); ``torch.distributed`` only carries the 128-byte rendezvous id (``init_comm``).  All ranks see the
  same commitments, feed the same transcript and return the same 768 bytes."""
from __future__ import annotations

import ctypes
from typing import Optional

from . import _lib
from .custom_gates import is_next_row
from .prover import Prover


def shard_range(n: int, rank: int, world: int):
    """Contiguous range [first, first+count) of rank `rank` out of `world` (the first n % world ranks get one
    extra item): the point-range cut of pb200_srs_commit_partial."""
    base, extra = divmod(n, world)
    first = rank * base + min(rank, extra)
    return first, base + (1 if rank < extra else 0)


def bucket_range(n_buckets: int, rank: int, world: int):
    """Bucket magnitudes [lo, hi) of rank `rank`: n_buckets // world each, starting at rank * (n_buckets // world) as
    the contiguous join (join_bucket_shards with nloc > 0) expects; the last rank also takes the n_buckets % world
    left over, so the ranges cover every bucket for any world size."""
    per = n_buckets // world
    return rank * per, n_buckets if rank == world - 1 else (rank + 1) * per


def combine_partials(parts: bytes, count: int):
    """Sum `count` XYZZ partial sums (128 bytes each, as produced by pb200_srs_commit_partial) into one affine
    point; returns (x||y little-endian bytes, is_identity).  Host arithmetic inside the library."""
    out = ctypes.create_string_buffer(64)
    ident = ctypes.c_int(0)
    _lib.check(_lib.lib().pb200_g1_combine_partials_host(parts, count, out, ctypes.byref(ident)))
    return out.raw, bool(ident.value)


def join_bucket_shards(sr: bytes, world: int, sets: int, nloc: int):
    """Host half of the sharded commitment's join: `sr` = [world][sets] (S, R) pairs of 2 x 128 bytes; returns a list
    of (x||y bytes, is_identity) per set.  nloc > 0: contiguous bucket ranges of that width; nloc == 0: strided
    ownership (rank rho owns the buckets world * k + rho), the layout the library's sharded commitments use."""
    out = ctypes.create_string_buffer(64 * sets)
    ident = (ctypes.c_int * sets)()
    _lib.check(_lib.lib().pb200_g1_join_bucket_shards_host(sr, world, sets, nloc, out, ident))
    return [(out.raw[64 * k:64 * k + 64], bool(ident[k])) for k in range(sets)]


def allgather_bytes(local: bytes, group=None, device=None) -> list:
    """All ranks contribute `local` (same length everywhere); returns the list of every rank's bytes.
    Uses a CUDA tensor (NCCL) when `device` is given, a CPU tensor (gloo) otherwise."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    t = torch.frombuffer(bytearray(local), dtype=torch.uint8)
    if device is not None:
        t = t.to(device)
    outs = [torch.empty_like(t) for _ in range(world)]
    dist.all_gather(outs, t, group=group)
    return [o.cpu().numpy().tobytes() for o in outs]


def broadcast_bytes(payload: Optional[bytes], size: int, src: int = 0, group=None, device=None) -> bytes:
    """Rank `src` sends `payload` (`size` bytes) to every rank of the group (NCCL when `device` is given, else gloo)."""
    import torch
    import torch.distributed as dist
    t = torch.zeros(size, dtype=torch.uint8)
    if dist.get_rank(group) == src:
        t = torch.frombuffer(bytearray(payload), dtype=torch.uint8).clone()
    if device is not None:
        t = t.to(device)
    dist.broadcast(t, src=dist.get_global_rank(group, src) if group is not None else src, group=group)
    return t.cpu().numpy().tobytes()


def init_comm(ctx: Optional[_lib.Context] = None, group=None) -> _lib.Context:
    """Give the library context its own NCCL communicator over the ranks of `group` (default: the world group):
    rank 0 draws the id, torch.distributed carries it, every rank joins.  Idempotent per context."""
    import torch
    import torch.distributed as dist
    ctx = ctx or _lib.default_context()
    if getattr(ctx, "comm_world", 1) > 1:
        return ctx
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    L = _lib.lib()
    uid = ctypes.create_string_buffer(128)
    if rank == 0:
        _lib.check(L.pb200_comm_unique_id(uid))
    device = torch.device("cuda", ctx.device) if dist.get_backend(group) == "nccl" else None
    raw = broadcast_bytes(uid.raw if rank == 0 else None, 128, 0, group, device)
    _lib.check(L.pb200_comm_init(ctx.handle, raw, rank, world))
    ctx.comm_rank, ctx.comm_world = rank, world
    return ctx


def comm_info(ctx: _lib.Context):
    """(rank, world, collectives issued, bytes received) of the context's communicator"""
    r, w = ctypes.c_int(), ctypes.c_int()
    c, b = ctypes.c_uint64(), ctypes.c_uint64()
    _lib.check(_lib.lib().pb200_comm_info(ctx.handle, ctypes.byref(r), ctypes.byref(w), ctypes.byref(c), ctypes.byref(b)))
    return r.value, w.value, c.value, b.value


class ShardedProver(Prover):
    """``Prover`` for one proof across the ranks of a process group: same constructor arguments, same methods,
    same bytes.  Every rank must make the same calls with the same inputs (the collectives inside are matched
    pairwise); the context needs a communicator (``init_comm``)."""
    _CREATE = "pb200_prover_create_sharded"
    sharded = True
    _CREATE_CUSTOM = "pb200_prover_create_custom_sharded"

    @classmethod
    def from_arrays(cls, setup, group_order, pk_arrays, group=None, ctx=None, custom=(), lookup=None, lookups=None,
                    shuffle=None):
        if lookup is not None or lookups is not None:
            raise ValueError("lookups are not available on the sharded prover (one GPU only)")
        if shuffle is not None:
            raise ValueError("shuffles are not available on the sharded prover (one GPU only)")
        custom = list(custom)
        if any(is_next_row(e) for e, _ in custom):
            raise ValueError("next-row custom gate terms are not available on the sharded prover (one GPU only)")
        init_comm(ctx or setup.ctx, group)
        return super().from_arrays(setup, group_order, pk_arrays, ctx=ctx, custom=custom)

    def __init__(self, setup, program, group=None):
        init_comm(setup.ctx, group)
        super().__init__(setup, program)

    def set_zk(self, enable: bool = True, blinders=None):
        """Zero-knowledge proving runs on one GPU only (``Prover.set_zk``)."""
        if enable:
            raise ValueError("zero-knowledge proving is not available on the sharded prover (one GPU only)")
        super().set_zk(False)

    def set_zk_lookup(self, enable: bool = True, blinders=None):
        """Zero-knowledge lookup proofs run on one GPU only (``Prover.set_zk_lookup``); so do lookups."""
        raise ValueError("zero-knowledge lookups are not available on the sharded prover (one GPU only)")

    def set_zk_shuffle(self, enable: bool = True, blinders=None):
        """Zero-knowledge shuffle proofs run on one GPU only (``Prover.set_zk_shuffle``); so do shuffles."""
        raise ValueError("zero-knowledge shuffles are not available on the sharded prover (one GPU only)")


# ------------------------------------------------------------------------------------------------
# operators (BASELINE.json metric: Fr-NTT elems/s and G1-MSM pts/s at 1/2/4/8 GPUs)
# ------------------------------------------------------------------------------------------------
def sharded_ntt(x_full, log_n: int, inverse: bool = False, ctx: Optional[_lib.Context] = None, out=None):
    """Distributed NTT of the length-2^log_n vector `x_full` (a CUDA tensor of N*32 bytes, present on every rank;
    only the rank's decimated part x[rank::world] is read).  Returns the FULL transform on every rank (a CUDA tensor
    [N, 32] uint8).  One NCCL allgather, issued by the library.  The context must carry a communicator."""
    import torch
    ctx = ctx or _lib.default_context()
    n = 1 << log_n
    if out is None:
        out = torch.empty((n, 32), dtype=torch.uint8, device=x_full.device)
    vp = ctypes.c_void_p
    _lib.check(_lib.lib().pb200_fr_ntt_sharded(ctx.handle, vp(x_full.data_ptr()), vp(out.data_ptr()), log_n,
                                               1 if inverse else 0))
    return out


def sharded_commit(setup, coeffs, m: int, montgomery: bool = False):
    """setup.py:66-72's MSM over device-resident coefficients `coeffs` (CUDA tensor, m*32 bytes, on every rank) with
    the buckets split over the ranks; returns ((x, y) ints or None).  One NCCL allgather of 256 bytes per rank."""
    out = ctypes.create_string_buffer(64)
    ident = ctypes.c_int()
    _lib.check(_lib.lib().pb200_srs_commit_coeffs_sharded(setup.ctx.handle, setup._srs, ctypes.c_void_p(coeffs.data_ptr()),
                                                          m, 1 if montgomery else 0, out, ctypes.byref(ident)))
    if ident.value:
        return None
    return int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little")
