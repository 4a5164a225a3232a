"""CPU: the two-level counting sort of the MSM's bucket entries (csrc/msm_sort.cuh), its kernel bodies run block by
block and phase by phase through csrc/host_selftest.cpp, checked against a plain grouping of the signed digits:
bucket b's entries at sorted[offsets[b] .. offsets[b] + counts[b]), offsets the exclusive prefix of the counts
(padded to even, pad slots 0xffffffff and the max count after the counts with `pad`)."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import plonk_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
DEFAULT_LB = 0xFFFFFFFF
STRIDED = lambda log_g: 0xFFFFFFFF - log_g  # hi argument of a strided shard of 2^log_g ranks


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "build", "host_selftest_sort.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in ("field.cuh", "curve.cuh", "msm_digits.cuh", "msm_bucket.cuh",
                                                    "msm_sort.cuh", "modinv.cuh", "ntt_shard.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    return ctypes.CDLL(out)


def _geometry(n, batch, c, fixed, lo, hi):
    W, half = (256 + c - 1) // c, 1 << (c - 1)
    if 0xFFFFFFF0 <= hi < 0xFFFFFFFF:
        log_g = 0xFFFFFFFF - hi
        own = lambda d: (d - 1) >> log_g if ((d - 1) & ((1 << log_g) - 1)) == lo else None
        nloc = half >> log_g
    else:
        hi = min(hi, half)
        own = lambda d: d - 1 - lo if lo <= d - 1 < hi else None
        nloc = hi - lo
    return W, nloc, own


def _reference(scalar_vecs, c, fixed, lo, hi):
    """bucket -> sorted list of entries, by walking the signed digits in Python"""
    n = len(scalar_vecs[0])
    W, nloc, own = _geometry(n, len(scalar_vecs), c, fixed, lo, hi)
    sets = len(scalar_vecs) if fixed else W
    groups = [[] for _ in range(sets * nloc)]
    for k, vec in enumerate(scalar_vecs):
        for i, s_ in enumerate(vec):
            carry = 0
            for w in range(W):
                d = ((s_ >> (w * c)) & ((1 << c) - 1)) + carry
                neg, carry = (1, 1) if d > 1 << (c - 1) else (0, 0)
                if neg:
                    d = (1 << c) - d
                if not d:
                    continue
                j = own(d)
                if j is None:
                    continue
                groups[(k if fixed else w) * nloc + j].append(((w * n if fixed else 0) + i) | (neg << 31))
    return [sorted(g) for g in groups]


def _sort(lib, scalar_vecs, c, fixed, lo, hi, pad, lb=DEFAULT_LB, T=16384, spb=0, bin_nt=512, chunk_nt=512):
    n, batch = len(scalar_vecs[0]), len(scalar_vecs)
    W, nloc, _ = _geometry(n, batch, c, fixed, lo, hi)
    nb = (batch if fixed else W) * nloc
    sc = (ctypes.c_uint32 * (8 * n * batch))()
    for k, vec in enumerate(scalar_vecs):
        for i, s_ in enumerate(vec):
            for w in range(8):
                sc[8 * (k * n + i) + w] = (s_ >> (32 * w)) & 0xFFFFFFFF
    cap = n * W * batch + nb
    counts = (ctypes.c_uint32 * (nb + 1))()
    off = (ctypes.c_uint32 * (nb + 1))()
    out = (ctypes.c_uint32 * cap)()
    got = lib.hs_msm_sort(sc, n, batch, c, 1 if fixed else 0, lo, hi, 1 if pad else 0, lb, T, spb, bin_nt,
                          chunk_nt, counts, off, out, cap)
    assert got == nb, (got, nb)
    return list(counts), list(off), list(out[:off[nb]])


def _check(lib, scalar_vecs, c, fixed, lo=0, hi=1 << 30, pad=False, **kw):
    ref = _reference(scalar_vecs, c, fixed, lo, hi)
    nb = len(ref)
    counts, off, out = _sort(lib, scalar_vecs, c, fixed, lo, hi, pad, **kw)
    assert counts[:nb] == [len(g) for g in ref]
    if pad:
        assert counts[nb] == max(len(g) for g in ref)
    run = 0
    for b, g in enumerate(ref):
        assert off[b] == run, b
        assert sorted(out[run:run + len(g)]) == g, b
        step = (len(g) + 1) & ~1 if pad else len(g)
        assert out[run + len(g):run + step] == [0xFFFFFFFF] * (step - len(g)), b
        run += step
    assert off[nb] == run == len(out)
    return ref


def _vectors(rng, n, batch, kind):
    if kind == "random":
        return [[rng.randrange(O.R_MOD) for _ in range(n)] for _ in range(batch)]
    if kind == "zero":
        return [[0] * n for _ in range(batch)]
    if kind == "equal":
        return [[rng.randrange(O.R_MOD)] * n for _ in range(batch)]
    assert kind == "half_zero"
    return [[rng.randrange(O.R_MOD) if rng.random() < 0.5 else 0 for _ in range(n)] for _ in range(batch)]


KINDS = ("random", "zero", "equal", "half_zero")


@pytest.mark.parametrize("kind", KINDS)
def test_msm_sort_generic_and_fixed_base(lib, kind):
    """batch 1-4 in fixed-base mode, generic mode, pad on and off, with the launch's bin width and chunk size and with
    narrow bins, short chunks and small blocks (several bin blocks, grid-stride chunks, bins of many chunks)"""
    rng = random.Random(KINDS.index(kind))
    small = dict(lb=1, T=7, spb=5, bin_nt=3, chunk_nt=5)
    for pad in (False, True):
        _check(lib, _vectors(rng, 37, 1, kind), 5, False, pad=pad)
        _check(lib, _vectors(rng, 37, 1, kind), 5, False, pad=pad, **small)
        for batch in (1, 2, 3, 4):
            _check(lib, _vectors(rng, 29, batch, kind), 4, True, pad=pad)
            _check(lib, _vectors(rng, 29, batch, kind), 4, True, pad=pad, **small)
            _check(lib, _vectors(rng, 29, batch, kind), 6, True, pad=pad, lb=0, T=3, spb=2, bin_nt=1, chunk_nt=2)


@pytest.mark.parametrize("kind", KINDS)
def test_msm_sort_shards(lib, kind):
    """contiguous bucket-range shards (a partial last bin when the range is not a multiple of the bin width) and
    strided shards: every rank's sort holds exactly its own buckets"""
    rng = random.Random(7 + len(kind))
    vecs = _vectors(rng, 31, 3, kind)
    for pad in (False, True):
        for lo, hi in ((0, 5), (3, 8), (5, 16), (1, 2)):
            _check(lib, vecs, 5, True, lo, hi, pad, lb=2, T=5, spb=4, bin_nt=2, chunk_nt=3)
            _check(lib, vecs, 5, True, lo, hi, pad)
        for log_g in (1, 2, 3):
            for r in range(1 << log_g):
                _check(lib, vecs, 5, True, r, STRIDED(log_g), pad, lb=1, T=4, spb=9, bin_nt=4, chunk_nt=3)
        _check(lib, vecs[:1], 5, False, 2, STRIDED(2), pad, lb=3, T=9, spb=1, bin_nt=2, chunk_nt=4)


def test_msm_sort_heavy_bin_and_default_width(lib):
    """a bin several chunks long (the short top window and equal scalars concentrate entries) at the launch's block
    sizes, and a wide window whose key count needs more than one key bit per bin (1280 bins of 64 buckets)"""
    rng = random.Random(3)
    vecs = [[5] * 300 + [rng.randrange(O.R_MOD) for _ in range(100)]]
    ref = _check(lib, vecs, 5, True, pad=True, T=64)
    assert max(len(g) for g in ref) > 4 * 64
    _check(lib, [[rng.randrange(O.R_MOD) for _ in range(150)]], 13, False, pad=False)
    _check(lib, [[rng.randrange(O.R_MOD) for _ in range(150)]], 13, False, pad=True, T=100, spb=40, bin_nt=32, chunk_nt=64)
