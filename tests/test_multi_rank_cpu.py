"""CPU, world_size 2 over gloo: the host-side logic of the multi-GPU joins (plonkathon_b200/parallel.py and the
library's host code): point-range and bucket-range MSM shards with one allgather of partial sums, the slab-sharded
NTT's join, the rendezvous broadcast.  The per-rank partial
MSMs are produced by the oracle here (no GPU in this container); on a GPU box the same code path runs with
NCCL and the CUDA MSM (tests/test_gpu_multi.py)."""
import os
import random
import socket

import pytest
import torch.multiprocessing as mp

from oracle import plonk_oracle as O

R256 = 1 << 256


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _xyzz_bytes(pt):
    """affine oracle point (or None) -> 128-byte XYZZ in Montgomery limbs, as the library stores partials"""
    if pt is None:
        return bytes(128)
    m = lambda v: (v * R256 % O.Q_MOD).to_bytes(32, "little")  # noqa: E731
    return m(pt[0]) + m(pt[1]) + m(1) + m(1)


def _worker(rank, world, port, n, seed, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from plonkathon_b200 import parallel
    rng = random.Random(seed)
    pts = [O.g1_multiply(O.G1, rng.randrange(1, O.R_MOD)) for _ in range(n)]
    sc = [rng.randrange(O.R_MOD) for _ in range(n)]
    if seed == 2:  # make the total cancel to the identity: second half negates the first
        h = n // 2
        pts = pts[:h] + pts[:h]
        sc = sc[:h] + [(-s) % O.R_MOD for s in sc[:h]]
    first, count = parallel.shard_range(n, rank, world)
    part = O.ec_lincomb_naive(list(zip(pts[first:first + count], sc[first:first + count]))) if count else None
    gathered = parallel.allgather_bytes(_xyzz_bytes(part))
    xy, ident = parallel.combine_partials(b"".join(gathered), world)
    got = None if ident else (int.from_bytes(xy[:32], "little"), int.from_bytes(xy[32:], "little"))
    q.put((rank, got == O.ec_lincomb_naive(list(zip(pts, sc))), ident))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("n,seed", [(9, 1), (8, 2)])
def test_sharded_msm_join_world2(n, seed):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, n, seed, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok, _ in res), res
    if seed == 2:
        assert all(ident for _, _, ident in res)


def test_shard_range_partitions():
    from plonkathon_b200.parallel import shard_range
    for n in (1, 7, 8, 1 << 20):
        for world in (1, 2, 3, 8):
            pos = 0
            for r in range(world):
                f, c = shard_range(n, r, world)
                assert f == pos
                pos += c
            assert pos == n


def test_bucket_range_covers_every_bucket():
    """contiguous bucket ranges for any world size: adjacent, from 0 to n_buckets, each starting at rank * (n // world)
    (the offset the contiguous join applies)"""
    from plonkathon_b200.parallel import bucket_range
    for nb in (1, 8, 2048, 1 << 20):
        for world in (1, 2, 3, 4, 5, 7, 8):
            cuts = [bucket_range(nb, r, world) for r in range(world)]
            assert cuts[0][0] == 0 and cuts[-1][1] == nb
            assert all(a[1] == b[0] for a, b in zip(cuts, cuts[1:]))
            assert all(lo == r * (nb // world) for r, (lo, _) in enumerate(cuts))


def _ntt_cpu_worker(rank, world, port, log_n, q):
    """the slab-sharded NTT of csrc/ntt_shard.cuh (pb200_fr_ntt_sharded) with the oracle standing in for the CUDA
    kernels: local transform of x[rank::world], join twiddle on the store, ONE allgather, a G-point DFT per element"""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from plonkathon_b200 import parallel
    n = 1 << log_n
    M = n // world
    rng = random.Random(3)
    x = [rng.randrange(O.R_MOD) for _ in range(n)]
    ok = True
    for inverse in (False, True):
        w = O.root_of_unity(n)
        if inverse:
            w = pow(w, -1, O.R_MOD)
        scale = pow(world, -1, O.R_MOD) if inverse else 1
        local = O.fft(x[rank::world], inv=inverse)         # step 1: local transform (carries 1/M when inverse)
        local = [v * pow(w, rank * k0, O.R_MOD) * scale % O.R_MOD for k0, v in enumerate(local)]  # fused store twiddle
        gathered = parallel.allgather_bytes(b"".join(v.to_bytes(32, "little") for v in local))   # step 2
        U = [[int.from_bytes(g[32 * t:32 * t + 32], "little") for t in range(M)] for g in gathered]
        wg = pow(w, M, O.R_MOD)
        full = [0] * n
        for k0 in range(M):                                 # step 3: length-G DFT over the rank index
            for k1 in range(world):
                full[k0 + M * k1] = sum(U[r][k0] * pow(wg, r * k1, O.R_MOD) for r in range(world)) % O.R_MOD
        ok = ok and full == O.fft(x, inv=inverse)
    q.put((rank, ok))
    dist.barrier()
    dist.destroy_process_group()


def test_slab_ntt_decomposition_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_ntt_cpu_worker, args=(r, 2, port, 8, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res), res


def _bucket_join_worker(rank, world, port, q):
    """the bucket-range MSM join (csrc/msm.cu, pb200_srs_commit_coeffs_sharded): every rank reduces its own range
    of signed-digit buckets to (S, R) = (sum B_j, sum (j+1) B_j), ONE allgather of 256 bytes per rank, and the
    library's host code adds sum_rho (R_rho + rho * nloc * S_rho).  Buckets are filled by the oracle here."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from plonkathon_b200 import parallel
    rng = random.Random(11)
    n, c = 10, 4
    half, W = 1 << (c - 1), (256 + c - 1) // c
    pts = [O.g1_multiply(O.G1, rng.randrange(1, O.R_MOD)) for _ in range(n)]
    sc = [rng.randrange(O.R_MOD) for _ in range(n - 2)] + [0, O.R_MOD - 1]
    # fixed-base layout: one bucket set shared by all windows, window w uses the point 2^(c w) P_i
    buckets = [None] * half
    for p, s_ in zip(pts, sc):
        carry, cur = 0, p
        for w in range(W):
            d = ((s_ >> (c * w)) & ((1 << c) - 1)) + carry
            carry = 0
            if d > half:
                d, carry = (1 << c) - d, 1
                if d:  # raw digit 2^c - 1 plus a carry folds to 0 with a carry out
                    buckets[d - 1] = O.g1_add(buckets[d - 1], O.g1_neg(cur))
            elif d:
                buckets[d - 1] = O.g1_add(buckets[d - 1], cur)
            cur = O.g1_multiply(cur, 1 << c)
    want = O.ec_lincomb_naive(list(zip(pts, sc)))
    ok = True
    lo, hi = parallel.bucket_range(half, rank, world)
    # contiguous ranges (operator level) and strided ownership (the library's sharded commitments): local bucket j
    for own, nloc in ((buckets[lo:hi], hi - lo), (buckets[rank::world], 0)):
        S = R = None
        for j, b in enumerate(own):
            S = O.g1_add(S, b)
            R = O.g1_add(R, O.g1_multiply(b, j + 1) if b else None)
        gathered = parallel.allgather_bytes(_xyzz_bytes(S) + _xyzz_bytes(R))
        (xy, ident), = parallel.join_bucket_shards(b"".join(gathered), world, 1, nloc)
        got = None if ident else (int.from_bytes(xy[:32], "little"), int.from_bytes(xy[32:], "little"))
        ok = ok and got == want
    q.put((rank, ok))
    dist.barrier()
    dist.destroy_process_group()


def test_bucket_range_msm_join_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_bucket_join_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res), res


def test_rendezvous_id_broadcast_world2():
    """parallel.broadcast_bytes: how the 128-byte communicator id reaches every rank (gloo here, NCCL on a GPU box)"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_bcast_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(ok for _, ok in res), res


def _bcast_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    import torch.distributed as dist
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from plonkathon_b200 import parallel
    payload = bytes(range(128))
    got = parallel.broadcast_bytes(payload if rank == 0 else None, 128, 0)
    q.put((rank, got == payload))
    dist.barrier()
    dist.destroy_process_group()
