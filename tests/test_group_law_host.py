"""CPU: the MSM's cheaper group law (csrc/field.cuh, csrc/curve.cuh) through csrc/host_selftest.cpp -- the dedicated
squaring, the lazily reduced products and differences on operands anywhere in [0, 2p), the sum of two products with
one reduction, and the XYZZ additions built from them, which must return the same limbs as the previous formulas
(canonical products throughout, two reductions for Y3)."""
import ctypes
import os
import random
import subprocess

import pytest

from oracle import plonk_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
R256 = 1 << 256
FIELDS = [(0, O.R_MOD), (1, O.Q_MOD)]
OP_MUL, OP_SQR, OP_MUL_LAZY, OP_SQR_LAZY, OP_SUB_LAZY, OP_NEG_LAZY, OP_IS_ZERO_LAZY = 2, 8, 11, 12, 13, 14, 15


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "build", "host_selftest_group_law.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in ("field.cuh", "curve.cuh", "msm_digits.cuh", "msm_bucket.cuh",
                                                    "msm_sort.cuh", "modinv.cuh", "ntt_shard.cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    return ctypes.CDLL(out)


def limbs(x, n=1):
    return (ctypes.c_uint32 * (8 * n))(*[(x >> (32 * i)) & 0xFFFFFFFF for i in range(8 * n)])


def unlimbs(buf, k=0):
    return sum(int(buf[8 * k + i]) << (32 * i) for i in range(8))


def fop(lib, field, op, a, b=0):
    out = (ctypes.c_uint32 * 8)()
    assert lib.hs_field_op(field, op, limbs(a), limbs(b), out) == 0
    return unlimbs(out)


def edge_values(p):
    """0, 1, p - 1, powers of two, limbs of all ones below p, and their lazy twins x + p"""
    canon = [0, 1, 2, p - 1, p - 2, (p - 1) // 2, (p + 1) // 2, R256 % p]
    canon += [1 << k for k in range(0, 254, 13)] + [(1 << k) - 1 for k in range(32, 254, 32)]
    canon += [(1 << 253) - 1, p >> 1, p - (1 << 128)]
    canon = [v for v in canon if v < p]
    return canon + [v + p for v in canon]


@pytest.mark.parametrize("field,p", FIELDS)
def test_sqr_matches_mul(lib, field, p):
    rng = random.Random(300 + field)
    rinv = pow(R256, -1, p)
    vals = edge_values(p)[: len(edge_values(p)) // 2] + [rng.randrange(p) for _ in range(2000)]
    for a in vals:
        sq = fop(lib, field, OP_SQR, a)
        assert sq == fop(lib, field, OP_MUL, a, a), hex(a)
        assert sq == a * a * rinv % p, hex(a)


@pytest.mark.parametrize("field,p", FIELDS)
def test_lazy_products_and_differences(lib, field, p):
    """inputs anywhere in [0, 2p): the right residue, and the result stays below 2p"""
    rng = random.Random(310 + field)
    rinv = pow(R256, -1, p)
    vals = edge_values(p) + [rng.randrange(2 * p) for _ in range(1500)]
    for i, a in enumerate(vals):
        b = vals[(i * 7 + 3) % len(vals)]
        r = fop(lib, field, OP_MUL_LAZY, a, b)
        assert r < 2 * p and r % p == a * b * rinv % p, (hex(a), hex(b))
        r = fop(lib, field, OP_SQR_LAZY, a)
        assert r < 2 * p and r % p == a * a * rinv % p, hex(a)
        r = fop(lib, field, OP_SUB_LAZY, a, b)
        assert r < 2 * p and r % p == (a - b) % p, (hex(a), hex(b))
        assert fop(lib, field, OP_IS_ZERO_LAZY, a) == (R256 % p if a % p == 0 else 0), hex(a)
        if a <= p:
            r = fop(lib, field, OP_NEG_LAZY, a)
            assert r <= p and r == p - a, hex(a)


@pytest.mark.parametrize("field,p", FIELDS)
def test_sum_of_two_products(lib, field, p):
    """redc(a b + c d) with one reduction, under its documented bound a b + c d < p R"""
    rng = random.Random(320 + field)
    rinv = pow(R256, -1, p)
    edge = edge_values(p)
    cases = []
    for _ in range(1500):
        # one factor of each product canonical, the other lazy (the group law's shape), or all canonical
        a, c = rng.choice([rng.randrange(2 * p), rng.choice(edge)]), rng.randrange(2 * p)
        b, d = rng.randrange(p), rng.choice([rng.randrange(p), rng.choice(edge) % p])
        cases.append((a, b, c, d))
    cases += [(2 * p - 1, p - 1, 2 * p - 1, p - 1), (0, 0, 0, 0), (p, p - 1, p, 1), (2 * p - 1, p, p - 1, p)]
    for a, b, c, d in cases:
        if a * b + c * d >= p * R256:
            continue
        out = (ctypes.c_uint32 * 8)()
        assert lib.hs_field_mul2(field, limbs(a), limbs(b), limbs(c), limbs(d), out) == 0
        r = unlimbs(out)
        assert r < 2 * p and r % p == (a * b + c * d) * rinv % p, (hex(a), hex(b), hex(c), hex(d))


def mont(x):
    return x * R256 % O.Q_MOD


def xyzz(pt):
    if pt is None:
        return limbs(0, 4)
    return limbs(mont(pt[0]) | (mont(pt[1]) << 256) | (mont(1) << 512) | (mont(1) << 768), 4)


def affine(pt):
    return limbs(mont(pt[0]) | (mont(pt[1]) << 256), 2)


def run(lib, fn, op, acc, other):
    out = (ctypes.c_uint32 * 32)()
    assert fn(op, acc, other, 0, out) == 0
    return out


def test_additions_match_previous_formulas(lib):
    """every addition and doubling, on random points with non-trivial ZZ, P + P, P + (-P) and identity operands,
    returns exactly the limbs the previous formulas return (all four coordinates canonical)"""
    rng = random.Random(330)
    pts = [O.g1_multiply(O.G1, rng.randrange(1, O.R_MOD)) for _ in range(10)]

    def both(op, acc, other):
        new, ref = run(lib, lib.hs_curve_op, op, acc, other), run(lib, lib.hs_curve_op_ref, op, acc, other)
        assert list(new) == list(ref), op
        for k in range(4):
            assert unlimbs(new, k) < O.Q_MOD
        return new

    for i, p in enumerate(pts):
        q = pts[(i + 3) % len(pts)]
        # accumulators with ZZ != 1: p + q, (p + q) + q, 2 (p + q)
        a1 = both(0, xyzz(p), affine(q))
        a2 = both(4, a1, affine(q))
        a3 = both(2, a1, limbs(0, 4))
        accs = [xyzz(p), a1, a2, a3, limbs(0, 4)]
        for acc in accs:
            for b in (p, q, O.g1_neg(p), O.g1_neg(q)):
                both(0, acc, affine(b))
                both(4, acc, affine(b))
            for other in accs:
                both(1, acc, other)
                both(5, acc, other)
            both(2, acc, limbs(0, 4))
        # P + P and P + (-P) with the accumulator in non-trivial coordinates: a1 + a1 (full add), a1 - a1
        both(1, a1, a1)
        both(5, a1, a1)
        neg_a1 = (ctypes.c_uint32 * 32)(*a1)
        neg_y = (-int(unlimbs(a1, 1))) % O.Q_MOD
        for k in range(8):
            neg_a1[8 + k] = (neg_y >> (32 * k)) & 0xFFFFFFFF
        for op in (1, 5):
            z = both(op, a1, neg_a1)
            assert unlimbs(z, 2) == 0  # the identity
        # the results also agree with the oracle's affine group law
        out = (ctypes.c_uint32 * 32)()
        assert lib.hs_curve_op(3, a2, limbs(0, 4), 0, out) == 0
        got = (unlimbs(out, 0) * pow(R256, -1, O.Q_MOD) % O.Q_MOD, unlimbs(out, 1) * pow(R256, -1, O.Q_MOD) % O.Q_MOD)
        assert got == O.g1_add(O.g1_add(p, q), q)
