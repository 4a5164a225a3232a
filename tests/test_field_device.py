"""GPU: Fr arithmetic of the compiled sm_90a code (the asm carry chains of csrc/field.cuh) at edge operands, checked
element by element against Python ints.

pb200_fr_vec_op (csrc/poly_ops.cu) runs ops 0-3 (a + b, a - b, a * b, a / b with inv(0) == 0), 4-6 (a + s, a - s,
a * s on every element), 7-8 (+ s, - s on element 0 only) and 9 (out[i] = a[(i + shift) mod n]); pb200_fr_to_mont /
pb200_fr_from_mont multiply by 2^256 and 2^-256.  Operands: every pair of about 40 edge values (0, 1, r - 1, (r +- 1) / 2,
2^256 mod r, all-ones limbs below r, powers of two, ...) plus random ones, at lengths that are not multiples of the
division kernel's 8-element chunks or of the 256-thread blocks, out of place and in place (d_out == d_a)."""
import ctypes
import random

import numpy as np
import pytest

from oracle import plonk_oracle as O
from tests.test_ntt_exact import empty_dev, ptr, to_dev, to_host

pytestmark = pytest.mark.gpu

R = O.R_MOD
R256 = 1 << 256
RINV = pow(R256, -1, R)
OP_ADD, OP_SUB, OP_MUL, OP_DIV, OP_ADD_S, OP_SUB_S, OP_MUL_S, OP_ADD_S0, OP_SUB_S0, OP_SHIFT = range(10)


def _edges():
    v = [0, 1, 2, 3, R - 1, R - 2, R - 3, (R - 1) // 2, (R + 1) // 2, R256 % R, R256 * R256 % R, RINV, R - R256 % R]
    v += [(1 << (32 * k)) - 1 for k in range(1, 8)]            # all-ones low limbs
    v += [1 << k for k in (31, 32, 63, 64, 127, 128, 191, 192, 224, 252, 253)]
    v += [R - (1 << 128), R - (1 << 32), (R >> 128 << 128) - 1, (R >> 32 << 32) - 1, R - (1 << 192) - 1,
          (1 << 253) - 1, (1 << 253) + 1, 0x30644E72E131A028FFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFF]
    out = sorted(set(x for x in v if 0 <= x < R))
    return out


EDGES = _edges()


def ints_to_arr(xs):
    return np.frombuffer(b"".join((x % R).to_bytes(32, "little") for x in xs), dtype=np.uint32).reshape(-1, 8).copy()


def arr_to_ints(a):
    raw = np.ascontiguousarray(a).tobytes()
    return [int.from_bytes(raw[32 * i:32 * i + 32], "little") for i in range(len(raw) // 32)]


def rand_ints(n, seed):
    """random elements below r with the edge values sprinkled in (every 5th element)"""
    rng = random.Random(seed)
    return [rng.choice(EDGES) if i % 5 == 0 else rng.randrange(R) for i in range(n)]


@pytest.fixture(scope="module")
def L():
    import plonkathon_b200  # noqa: F401
    from plonkathon_b200 import _lib
    return _lib


def vec_op(L, op, a, b=None, s=None, shift=0, in_place=False):
    """one pb200_fr_vec_op call on Python-int vectors (or an (n, 8) uint32 array a); returns the output as Python
    ints, or as an array when a is one"""
    n = len(a)
    d_a = to_dev(a if isinstance(a, np.ndarray) else ints_to_arr(a))
    b_arr = ints_to_arr(b) if b is not None else None
    d_b = to_dev(b_arr) if b is not None else None
    d_out = d_a if in_place else empty_dev(n)
    h_s = (s % R).to_bytes(32, "little") if s is not None else None
    L.check(L.lib().pb200_fr_vec_op(L.default_context().handle, op, ptr(d_a), ptr(d_b) if d_b is not None else None,
                                    h_s, ptr(d_out), n, shift))
    got = to_host(d_out, L) if isinstance(a, np.ndarray) else arr_to_ints(to_host(d_out, L))
    if b is not None:
        assert np.array_equal(to_host(d_b, L), b_arr), "the second operand changed"
    return got


def mont(L, a, inverse, in_place=False):
    d_a = to_dev(ints_to_arr(a))
    d_out = d_a if in_place else empty_dev(len(a))
    fn = L.lib().pb200_fr_from_mont if inverse else L.lib().pb200_fr_to_mont
    L.check(fn(L.default_context().handle, ptr(d_a), ptr(d_out), len(a)))
    return arr_to_ints(to_host(d_out, L))


def quotients(a, b):
    """a_i / b_i with inv(0) == 0, by one batch inversion (Montgomery's trick) over the nonzero b_i"""
    pref, run = [], 1
    for y in b:
        pref.append(run)
        if y:
            run = run * y % R
    inv, out = pow(run, -1, R), [0] * len(b)
    for i in range(len(b) - 1, -1, -1):
        if b[i]:
            out[i] = a[i] * inv % R * pref[i] % R
            inv = inv * b[i] % R
    return out


def expect(op, a, b=None, s=None, shift=0):
    if op == OP_ADD:
        return [(x + y) % R for x, y in zip(a, b)]
    if op == OP_SUB:
        return [(x - y) % R for x, y in zip(a, b)]
    if op == OP_MUL:
        return [x * y % R for x, y in zip(a, b)]
    if op == OP_DIV:
        return quotients(a, b)
    if op == OP_ADD_S:
        return [(x + s) % R for x in a]
    if op == OP_SUB_S:
        return [(x - s) % R for x in a]
    if op == OP_MUL_S:
        return [x * s % R for x in a]
    if op in (OP_ADD_S0, OP_SUB_S0):
        return [((a[0] + s if op == OP_ADD_S0 else a[0] - s) % R)] + list(a[1:])
    n = len(a)
    return [a[(i + shift) % n] for i in range(n)]


def first_bad(got, want):
    bad = [i for i, (g, w) in enumerate(zip(got, want)) if g != w]
    return (len(bad), bad[:4]) if bad or len(got) != len(want) else None


# ------------------------------------------------------------------ every pair of edge values
@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
@pytest.mark.parametrize("op", [OP_ADD, OP_SUB, OP_MUL, OP_DIV])
def test_binary_ops_edge_cross_product(L, op, in_place):
    """ops 0-3 on the full cross product of the edge set (n = |E|^2, not a multiple of 8 or of 256): 0 and r - 1 meet
    every operand, every sum and difference that wraps, and x / 0 == 0"""
    a = [x for x in EDGES for _ in EDGES]
    b = [y for _ in EDGES for y in EDGES]
    assert len(a) % 8 and len(a) % 256
    got = vec_op(L, op, a, b, in_place=in_place)
    assert first_bad(got, expect(op, a, b)) is None, (op, first_bad(got, expect(op, a, b)))


@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
@pytest.mark.parametrize("op", [OP_ADD_S, OP_SUB_S, OP_MUL_S, OP_ADD_S0, OP_SUB_S0])
def test_scalar_ops_every_edge_scalar(L, op, in_place):
    """ops 4-8 with every edge value as the scalar, on a vector of every edge value followed by random elements"""
    a = EDGES + rand_ints(257 - len(EDGES), 40 + op)
    for s in EDGES:
        got = vec_op(L, op, a, s=s, in_place=in_place)
        assert first_bad(got, expect(op, a, s=s)) is None, (op, hex(s), first_bad(got, expect(op, a, s=s)))


@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
def test_montgomery_conversion_edges(L, in_place):
    """pb200_fr_to_mont / pb200_fr_from_mont: x 2^256 and x 2^-256 mod r for every edge value, and back"""
    a = EDGES + rand_ints(100, 7)
    m = mont(L, a, False, in_place)
    assert m == [x * R256 % R for x in a]
    assert mont(L, a, True, in_place) == [x * RINV % R for x in a]
    assert mont(L, m, True, in_place) == a


# ------------------------------------------------------------------ lengths around the chunk and block sizes
SIZES = [1, 7, 8, 9, 255, 257, len(EDGES) ** 2, (1 << 20) + 5]


@pytest.mark.parametrize("n", SIZES)
def test_every_op_at_odd_lengths(L, n):
    """every op at n elements, random operands with edges sprinkled in and about one divisor in 16 zero; the
    last element (where a short tail block or chunk ends) and element 0 (ops 7-8) are in every check"""
    a, b = rand_ints(n, 1000 + n), rand_ints(n, 2000 + n)
    rng = random.Random(n)
    for i in range(n):
        if rng.random() < 1 / 16:
            b[i] = 0
    s = rng.choice(EDGES[1:])
    for op in range(OP_SHIFT):
        in_place = op % 2 == 1
        two = op <= OP_DIV
        got = vec_op(L, op, a, b if two else None, None if two else s, in_place=in_place)
        want = expect(op, a, b if two else None, s)
        assert first_bad(got, want) is None, (n, op, first_bad(got, want))
    a_arr = ints_to_arr(a)
    for shift in sorted({0, 1, n - 1, n, n + 3, 2 * n + 1}):
        assert np.array_equal(vec_op(L, OP_SHIFT, a_arr, shift=shift), np.roll(a_arr, -(shift % n), axis=0)), (n, shift)
    m = mont(L, a, False)
    assert m == [x * R256 % R for x in a]
    assert mont(L, m, True, in_place=True) == a


def test_shift_refuses_in_place(L):
    from plonkathon_b200._lib import PlonkB200Error
    with pytest.raises(PlonkB200Error, match="in place"):
        vec_op(L, OP_SHIFT, [1, 2, 3], shift=1, in_place=True)
    assert vec_op(L, OP_ADD, [1, 2, 3], [R - 1, R - 2, R - 3]) == [0, 0, 0]  # the context still works


# ------------------------------------------------------------------ division: zero divisors inside the shared inversion
@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
@pytest.mark.parametrize("n", [9, 255, 257, 1000, 4096, (1 << 20) + 5])
def test_division_zero_divisors_in_chunks(L, n, in_place):
    """k_vec_div shares one inversion between the 8 elements t, t + T, ..., t + 7T (T = ceil(n / 8)): zero divisors
    at the first, a middle and the last slot of a chunk, and one chunk made only of zeros; every other quotient of
    those chunks must survive"""
    T = (n + 7) // 8
    a, b = rand_ints(n, 3000 + n), rand_ints(n, 4000 + n)
    b = [y if y else 1 for y in b]  # zero divisors only where placed below
    slots = lambda t: [t + k * T for k in range(8) if t + k * T < n]  # noqa: E731
    for t, where in ((0, "first"), (T // 3, "last"), (T // 2, "middle"), (T - 1, "first"), (T - 1, "last")):
        s = slots(t)
        b[s[{"first": 0, "middle": len(s) // 2, "last": -1}[where]]] = 0
    for i in slots(T // 4 if T > 4 else T - 1):
        b[i] = 0  # a chunk of zero divisors only
    got = vec_op(L, OP_DIV, a, b, in_place=in_place)
    want = expect(OP_DIV, a, b)
    assert first_bad(got, want) is None, (n, first_bad(got, want))
