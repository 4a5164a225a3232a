"""CPU: the limb-level field / curve arithmetic of csrc/field.cuh + csrc/curve.cuh, compiled for
the host (PTX carry primitives replaced by their emulation) and checked against Python ints and
the oracle's affine group law.  This is the same C++ the CUDA kernels instantiate."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import plonk_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
R256 = 1 << 256


def _build(name, *defines):
    out = os.path.join(ROOT, "build", name)
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in ("field.cuh", "curve.cuh", "msm_digits.cuh", "msm_bucket.cuh", "modinv.cuh", "ntt_shard.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", *defines, "-x", "c++", src,
                               "-I", CSRC, "-o", out])
    return ctypes.CDLL(out)


@pytest.fixture(scope="module")
def lib():
    return _build("host_selftest.so")


@pytest.fixture(scope="module")
def fast_lib():
    """the same source built as the library builds its host code: with -DPB_HOST_FAST_MUL, fp_mul, fp_mul_lazy,
    fp_sqr_lazy and fp_mul2_lazy run fp_mul_host64 (4 x 64-bit CIOS) on the host, the arithmetic of the pairing,
    challenge reduction and the affine conversion of MSM results"""
    return _build("host_selftest_fast_mul.so", "-DPB_HOST_FAST_MUL")


def limbs(x, n=1):
    return (ctypes.c_uint32 * (8 * n))(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(8 * n)])


def unlimbs(buf, k=0):
    return sum(int(buf[8 * k + i]) << (32 * i) for i in range(8))


def fop(lib, field, op, a, b=0):
    out = (ctypes.c_uint32 * 8)()
    assert lib.hs_field_op(field, op, limbs(a), limbs(b), out) == 0
    return unlimbs(out)


EDGE = [0, 1, 2, 3, 0xFFFFFFFF, 1 << 32, (1 << 64) - 1, (1 << 128) + 1, (1 << 224) - 1]


@pytest.mark.parametrize("field,p", [(0, O.R_MOD), (1, O.Q_MOD)])
def test_field_ops(lib, field, p):
    rng = random.Random(field)
    vals = EDGE + [p - 1, p - 2, (p - 1) // 2, R256 % p, (R256 * R256) % p] + \
        [rng.randrange(p) for _ in range(200)]
    rinv = pow(R256, -1, p)
    for i, a in enumerate(vals):
        b = vals[(i * 7 + 3) % len(vals)]
        assert fop(lib, field, 0, a, b) == (a + b) % p
        assert fop(lib, field, 1, a, b) == (a - b) % p
        assert fop(lib, field, 2, a, b) == a * b * rinv % p
        assert fop(lib, field, 8, a) == a * a * rinv % p
        assert fop(lib, field, 3, a) == (-a) % p
        assert fop(lib, field, 7, a) == 2 * a % p
        assert fop(lib, field, 5, a) == a * R256 % p
        assert fop(lib, field, 6, a) == a * rinv % p
    for a in vals[:40]:
        am = a * R256 % p
        inv = fop(lib, field, 4, am)
        assert inv == (pow(a, -1, p) * R256 % p if a else 0)


def mont(x):
    return x * R256 % O.Q_MOD


def unmont(x):
    return x * pow(R256, -1, O.Q_MOD) % O.Q_MOD


def xyzz(lib, pt):
    """affine int point (or None) -> XYZZ limbs buffer"""
    if pt is None:
        return limbs(0, 4)
    v = mont(pt[0]) | (mont(pt[1]) << 256) | (mont(1) << 512) | (mont(1) << 768)
    return limbs(v, 4)


def to_affine(lib, acc):
    out = (ctypes.c_uint32 * 32)()
    inf = lib.hs_curve_op(3, acc, limbs(0, 4), 0, out)
    return None if inf else (unmont(unlimbs(out, 0)), unmont(unlimbs(out, 1)))


def test_curve_ops(lib):
    rng = random.Random(5)
    G = O.G1
    pts = [O.g1_multiply(G, rng.randrange(1, O.R_MOD)) for _ in range(12)]
    for i, p in enumerate(pts):
        q = pts[(i + 1) % len(pts)]
        for a, b in ((p, q), (p, p), (p, O.g1_neg(p)), (None, q), (p, None)):
            acc = xyzz(lib, a)
            out = (ctypes.c_uint32 * 32)()
            if b is not None:  # mixed add
                bb = limbs(mont(b[0]) | (mont(b[1]) << 256), 2)
                lib.hs_curve_op(0, acc, bb, 0, out)
                assert to_affine(lib, out) == O.g1_add(a, b)
                out_u = (ctypes.c_uint32 * 32)()
                lib.hs_curve_op(4, acc, bb, 0, out_u)  # SIMT-uniform variant
                assert to_affine(lib, out_u) == O.g1_add(a, b)
            lib.hs_curve_op(1, acc, xyzz(lib, b), 0, out)  # full add
            assert to_affine(lib, out) == O.g1_add(a, b)
            out_u2 = (ctypes.c_uint32 * 32)()
            lib.hs_curve_op(5, acc, xyzz(lib, b), 0, out_u2)  # select-based full add
            assert to_affine(lib, out_u2) == O.g1_add(a, b)
        # chains with non-trivial ZZ: ((p+q)+q)+(p+q) etc.
        acc = xyzz(lib, p)
        bb = limbs(mont(q[0]) | (mont(q[1]) << 256), 2)
        o1 = (ctypes.c_uint32 * 32)()
        lib.hs_curve_op(0, acc, bb, 0, o1)
        o2 = (ctypes.c_uint32 * 32)()
        lib.hs_curve_op(0, o1, bb, 0, o2)
        exp = O.g1_add(O.g1_add(p, q), q)
        assert to_affine(lib, o2) == exp
        o3 = (ctypes.c_uint32 * 32)()
        lib.hs_curve_op(1, o2, o1, 0, o3)
        assert to_affine(lib, o3) == O.g1_add(exp, O.g1_add(p, q))
        o3u = (ctypes.c_uint32 * 32)()
        lib.hs_curve_op(5, o2, o1, 0, o3u)
        assert to_affine(lib, o3u) == to_affine(lib, o3)
        o4 = (ctypes.c_uint32 * 32)()
        lib.hs_curve_op(1, o3, o3, 0, o4)  # projective doubling through add
        assert to_affine(lib, o4) == O.g1_double(O.g1_add(exp, O.g1_add(p, q)))
        o5 = (ctypes.c_uint32 * 32)()
        lib.hs_curve_op(2, o3, limbs(0, 4), 0, o5)
        assert to_affine(lib, o5) == to_affine(lib, o4)


@pytest.mark.parametrize("log_g", [1, 2, 3])
def test_sharded_ntt_join_dft(lib, log_g):
    """csrc/ntt_shard.cuh small_dft: the G-point DFT over the rank index at the join of the slab-sharded NTT, as the
    kernel instantiates it (bit-reversed input, radix-2 butterflies in registers), against the definition -- forward and
    inverse roots"""
    rng = random.Random(log_g)
    p, G = O.R_MOD, 1 << log_g
    mont = lambda v: v * R256 % p  # noqa: E731
    for w in (pow(O.root_of_unity(64), 64 // G, p), pow(O.root_of_unity(64), -(64 // G), p)):
        x = [rng.randrange(p) for _ in range(G)]
        xb = (ctypes.c_uint32 * (8 * G))(*[(mont(v) >> (32 * i)) & 0xFFFFFFFF for v in x for i in range(8)])
        tw = (ctypes.c_uint32 * 32)(*[(mont(pow(w, k, p)) >> (32 * i)) & 0xFFFFFFFF for k in range(4) for i in range(8)])
        out = (ctypes.c_uint32 * (8 * G))()
        assert lib.hs_small_dft(log_g, xb, tw, out) == 0
        got = [unlimbs(out, k) * pow(R256, -1, p) % p for k in range(G)]
        assert got == [sum(x[r] * pow(w, r * k, p) for r in range(G)) % p for k in range(G)]


def test_msm_signed_digit_slicing(lib):
    """csrc/msm_digits.cuh: for every window size the MSM can pick, the signed digits reconstruct the scalar,
    stay within [-2^(c-1), 2^(c-1)] and leave no carry -- including the field's edge values"""
    rng = random.Random(21)
    scalars = [0, 1, 2, O.R_MOD - 1, O.R_MOD - 2, (1 << 253), (1 << 254) - 1 - ((1 << 254) - O.R_MOD) - 1,
               (1 << 200) - 1, int("55" * 31, 16), int("aa" * 31, 16) % O.R_MOD] + [rng.randrange(O.R_MOD) for _ in range(60)]
    for c in range(4, 23):
        for s_ in scalars:
            digits = (ctypes.c_int32 * 64)()
            nw = ctypes.c_uint32(0)
            carry = lib.hs_msm_digits(limbs(s_), c, digits, ctypes.byref(nw))
            assert carry == 0, (c, hex(s_))
            assert nw.value == (256 + c - 1) // c
            ds = [digits[w] for w in range(nw.value)]
            assert all(abs(d) <= 1 << (c - 1) for d in ds), (c, hex(s_))
            assert sum(d << (c * w) for w, d in enumerate(ds)) == s_, (c, hex(s_))


def _pts_buf(points):
    buf = (ctypes.c_uint32 * (16 * len(points)))()
    for i, (x, y) in enumerate(points):
        for k in range(8):
            buf[16 * i + k] = (x >> (32 * k)) & 0xFFFFFFFF
            buf[16 * i + 8 + k] = (y >> (32 * k)) & 0xFFFFFFFF
    return buf


def _msm_pipeline(lib, points, scalar_vecs, c, fixed, lo, hi, B, g0):
    n, batch = len(points), len(scalar_vecs)
    sc = (ctypes.c_uint32 * (8 * n * batch))()
    for k, vec in enumerate(scalar_vecs):
        for i, s_ in enumerate(vec):
            for w in range(8):
                sc[8 * (k * n + i) + w] = (s_ >> (32 * w)) & 0xFFFFFFFF
    out = (ctypes.c_uint32 * (16 * batch))()
    inf = (ctypes.c_uint8 * batch)()
    rounds = lib.hs_msm_pipeline(_pts_buf(points), n, sc, batch, c, 1 if fixed else 0, lo, hi, B, g0, out, inf)
    assert rounds >= 1, rounds
    return [None if inf[k] else (unlimbs(out, 2 * k), unlimbs(out, 2 * k + 1)) for k in range(batch)], rounds


def _oracle_msm(points, scalars):
    acc = None
    for pt, s_ in zip(points, scalars):
        if s_ % O.R_MOD:
            acc = O.g1_add(acc, O.g1_multiply(pt, s_ % O.R_MOD))
    return acc


def test_msm_bucket_pipeline_on_host(lib):
    """csrc/msm_bucket.cuh + msm_digits.cuh: the whole MSM bucket pipeline (signed digits, padded counting sort, rounds
    of batched affine additions with the safegcd inversion, recursive bucket reduction, bucket-range shards), every
    GPU thread body run in a loop on the CPU, against the oracle's group law (curve.py:38-44 semantics)."""
    rng = random.Random(99)
    base = [O.g1_multiply(O.G1, rng.randrange(1, O.R_MOD)) for _ in range(12)]
    # repeated and opposite points: same-bucket collisions exercise doubling, P + (-P) and identities in later rounds
    points = base + [base[0], base[0], O.g1_neg(base[1]), base[1], base[2], base[2], base[2], O.g1_neg(base[2])]
    n = len(points)
    edge = [0, 1, 2, O.R_MOD - 1, O.R_MOD - 2, (1 << 253) + 5, 15, 16, 17, (1 << 128) - 1]
    rand = lambda: [rng.choice(edge) if rng.random() < 0.3 else rng.randrange(O.R_MOD) for _ in range(n)]
    # generic mode (one bucket set per window), several blockings
    for c, B, g0 in ((4, 2, 2), (4, 5, 4), (5, 128, 16), (3, 3, 2)):
        sc = rand()
        got, _ = _msm_pipeline(lib, points, [sc], c, False, 0, 1 << 30, B, g0)
        assert got[0] == _oracle_msm(points, sc), (c, B, g0)
    # all scalars equal: every window has one heavy bucket (cnt = n = 20 -> 5 rounds), with the collisions above
    for s_ in (1, 7, O.R_MOD - 1, 0x1111111111111111111111111111111111111111111111111111111111111111 % O.R_MOD):
        got, rounds = _msm_pipeline(lib, points, [[s_] * n], 4, False, 0, 1 << 30, 3, 4)
        assert got[0] == _oracle_msm(points, [s_] * n), hex(s_)
        assert rounds == 5
    # fixed-base mode: batched scalar vectors share the window table and one bucket set each
    vecs = [rand(), rand(), [3] * n]
    expect = [_oracle_msm(points, v) for v in vecs]
    got, _ = _msm_pipeline(lib, points, vecs, 5, True, 0, 1 << 30, 7, 4)
    assert got == expect
    # bucket-range shards (multi-GPU MSM join): the partial sums of disjoint ranges add up to the full result
    for cuts in ((0, 16), (0, 5, 16), (0, 1, 2, 9, 16), (0, 4, 8, 12, 16)):
        acc = [None] * len(vecs)
        for lo, hi in zip(cuts[:-1], cuts[1:]):
            part, _ = _msm_pipeline(lib, points, vecs, 5, True, lo, hi, 4, 2)
            acc = [O.g1_add(a, p) for a, p in zip(acc, part)]
        assert acc == expect, cuts
    # wide windows: 4096 buckets per window, two block-level chunks and a second block level in the reduction
    sc = rand()
    got, _ = _msm_pipeline(lib, points, [sc], 13, False, 0, 1 << 30, 16, 2)
    assert got[0] == _oracle_msm(points, sc)
    # strided shards (what the communicator path uses: rank r owns the buckets G k + r, so the buckets a short top
    # window concentrates on spread over all ranks): the partial sums G R + (r + 1 - G) S add up to the full result
    for log_g in (1, 2, 3):
        acc = [None] * len(vecs)
        for r in range(1 << log_g):
            part, _ = _msm_pipeline(lib, points, vecs, 5, True, r, 0xFFFFFFFF - log_g, 4, 2)
            acc = [O.g1_add(a, p) for a, p in zip(acc, part)]
        assert acc == expect, log_g
    # an empty result: all scalars zero
    got, _ = _msm_pipeline(lib, points, [[0] * n], 4, False, 0, 1 << 30, 4, 4)
    assert got == [None]
    # one bucket with more than 2^12 entries: the rounds past PB_AFF_GRID_ROUNDS (k_aff_tail's share on the GPU)
    many, cur = [], O.G1
    for _ in range(4200):
        many.append(cur)
        cur = O.g1_add(cur, O.G1)  # i * G: distinct points
    got, rounds = _msm_pipeline(lib, many, [[5] * len(many)], 4, False, 0, 1 << 30, 16, 16)
    assert rounds == 13
    assert got[0] == O.g1_multiply(O.G1, 5 * (4200 * 4201 // 2))


@pytest.mark.parametrize("field,p", [(0, O.R_MOD), (1, O.Q_MOD)])
def test_safegcd_inverse(lib, field, p):
    """csrc/modinv.cuh: inversion by batches of 30 Bernstein-Yang division steps on signed 30-bit limbs -- plain
    integers against pow(x, -1, p), and the Montgomery-form wrapper against the Fermat fp_inv it is meant to replace"""
    rng = random.Random(40 + field)
    vals = EDGE + [p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R256 % p, 1 << 253, (1 << 253) + 1, 3 << 252 if (3 << 252) < p else 5,
                   (1 << 30) - 1, 1 << 30, (1 << 60) + 1, p - (1 << 30), p - (1 << 200)]
    vals += [rng.randrange(p) for _ in range(3000)]
    vals += [rng.randrange(1 << k) for k in range(1, 254, 7) for _ in range(4)]
    for a in vals:
        a %= p
        assert fop(lib, field, 10, a) == (pow(a, -1, p) if a else 0), a
    for a in vals[:400]:
        a %= p
        assert fop(lib, field, 9, a) == fop(lib, field, 4, a), a


# ------------------------------------------------------------------ the fast host multiply (fp_mul_host64)
def _fast_mul_checks():
    from tests import test_group_law_host as GL
    return {"field_ops": test_field_ops, "safegcd_inverse": test_safegcd_inverse, "sqr_matches_mul": GL.test_sqr_matches_mul,
            "lazy_products": GL.test_lazy_products_and_differences, "sum_of_two_products": GL.test_sum_of_two_products}


@pytest.mark.parametrize("check", sorted(_fast_mul_checks()))
@pytest.mark.parametrize("field,p", [(0, O.R_MOD), (1, O.Q_MOD)])
def test_fast_host_mul(fast_lib, check, field, p):
    """the edge-value checks of the limb build, run against the -DPB_HOST_FAST_MUL build (its lazy results are
    canonical, so the < 2p bounds hold as well)"""
    _fast_mul_checks()[check](fast_lib, field, p)
