"""GPU: the Fr transforms checked exactly at every size from 2^0 to 2^24, through the one-, two- and three-pass plans
(ntt.cu build_plan: one pass up to 2^11, two up to 2^22, three from 2^23).

A whole output vector is checked in O(n) host time by a polynomial identity at one random point z off the domain:
forward, eval_lagrange(NTT(x), z) == eval_coeffs(x, z); inverse, eval_coeffs(iNTT(x), z) == eval_lagrange(x, z).  If
the output is wrong anywhere, the two sides differ as polynomials of degree < n, so they agree at a random z with
probability at most n / r < 2^-225.  Both sides come from the C restatement (oracle/c/plonk_oracle.c).
PB200_TEST_2P24=1 adds 2^25 and 2^26."""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import c_oracle as C
from oracle import plonk_oracle as O

pytestmark = pytest.mark.gpu

R = O.R_MOD
COSET = 5  # the prover's fixed coset g * <w_4n> (prover.cu)
_rng = random.Random(20261017)
Z = _rng.randrange(2, R)
OFFSET = _rng.randrange(2, R)
assert pow(Z, 1 << 28, R) != 1  # z is off every domain the transforms use, and so are g z and z / g
BIG = os.environ.get("PB200_TEST_2P24") == "1"
big_only = pytest.mark.skipif(not BIG, reason="opt-in (PB200_TEST_2P24=1): 2^25 and 2^26 points, minutes of host work")


@pytest.fixture(scope="module")
def L():
    import plonkathon_b200  # noqa: F401
    from plonkathon_b200 import _lib
    return _lib


def fr_bytes(x):
    return (int(x) % R).to_bytes(32, "little")


def row(x):
    return np.frombuffer(fr_bytes(x), dtype=np.uint32)


def random_fr(n, seed):
    """n canonical scalars as (n, 8) uint32 limbs: uniform below 2^252, with r - 1 and 0 sprinkled in"""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint32)
    a[:, 7] &= 0x0FFFFFFF
    if n >= 4:
        a[rng.integers(0, n, size=max(1, n // 64))] = row(R - 1)
        a[n - 1] = row(R - 1)
        a[n // 2] = 0
    return a


def to_dev(a):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).cuda()
    torch.cuda.synchronize()
    return t


def empty_dev(n):
    import torch
    return torch.empty((n, 8), dtype=torch.int32, device="cuda")


def ptr(t):
    return ctypes.c_void_p(t.data_ptr())


def to_host(t, L):
    L.default_context().sync()
    return t.cpu().numpy().view(np.uint32).reshape(-1, 8)


def ntt(L, x, log_n, inverse, in_place=False):
    d_in = to_dev(x)
    d_out = d_in if in_place else empty_dev(1 << log_n)
    L.check(L.lib().pb200_fr_ntt(L.default_context().handle, ptr(d_in), ptr(d_out), log_n, 1 if inverse else 0))
    return to_host(d_out, L)


# ------------------------------------------------------------------ every size, random inputs
@pytest.mark.parametrize("log_n", list(range(0, 25)) + [pytest.param(25, marks=big_only),
                                                        pytest.param(26, marks=big_only)])
def test_ntt_every_size_exact(L, log_n):
    n = 1 << log_n
    x = random_fr(n, 1000 + log_n)
    y = ntt(L, x, log_n, False)
    assert C.eval_lagrange(y, Z) == C.eval_coeffs(x, Z), "forward NTT wrong at 2^%d" % log_n
    u = ntt(L, x, log_n, True)
    assert C.eval_coeffs(u, Z) == C.eval_lagrange(x, Z), "inverse NTT wrong at 2^%d" % log_n
    if log_n == 23:  # the first three-pass size (8/8/7), also element by element against the C FFT
        assert np.array_equal(y.view(np.uint8), C.fft(x.view(np.uint8).reshape(n, 32), False))


# ------------------------------------------------------------------ edge inputs on each side of a pass boundary
def _check_const(out, value, first=None):
    """every element == value, except element 0 == first when given"""
    if first is not None:
        assert np.array_equal(out[0], row(first)), "element 0"
        out = out[1:]
    assert np.all(out == row(value)[None, :]), "not the constant %d everywhere" % value


@pytest.mark.parametrize("in_place", [False, True], ids=["out_of_place", "in_place"])
@pytest.mark.parametrize("log_n", [11, 12, 22, 23, 24])
def test_ntt_edge_inputs_exact(L, log_n, in_place):
    """all zeros, all r - 1, a delta at 0 and at n - 1, forward and inverse, with d_out == d_in or apart: closed forms
    (constants, or the geometric series of w^-k and w^k / n checked at z)"""
    n = 1 << log_n
    n_inv = pow(n, -1, R)
    w = O.root_of_unity(n)
    zeros = np.zeros((n, 8), dtype=np.uint32)
    _check_const(ntt(L, zeros, log_n, False, in_place), 0)
    _check_const(ntt(L, zeros, log_n, True, in_place), 0)
    minus_one = np.tile(row(R - 1), (n, 1))
    _check_const(ntt(L, minus_one, log_n, False, in_place), 0, first=-n)  # -1 at every point: -n at frequency 0
    _check_const(ntt(L, minus_one, log_n, True, in_place), 0, first=R - 1)  # the constant polynomial -1
    d0 = zeros.copy()
    d0[0, 0] = 1
    _check_const(ntt(L, d0, log_n, False, in_place), 1)
    _check_const(ntt(L, d0, log_n, True, in_place), n_inv)
    dl = zeros.copy()
    dl[n - 1, 0] = 1
    zn1 = (pow(Z, n, R) - 1) % R
    y = ntt(L, dl, log_n, False, in_place)  # y_k = w^-k
    assert np.array_equal(y[0], row(1))
    assert C.eval_coeffs(y, Z) == zn1 * pow(Z * pow(w, -1, R) - 1, -1, R) % R
    u = ntt(L, dl, log_n, True, in_place)  # u_k = w^k / n
    assert np.array_equal(u[0], row(n_inv))
    assert C.eval_coeffs(u, Z) == zn1 * n_inv % R * pow(Z * w - 1, -1, R) % R


# ------------------------------------------------------------------ the strided transform (slab-sharded NTT's local step)
_DECIMATED = [(log_m, s, o) for log_m in (10, 12, 21) for s in (1, 2, 4, 8) for o in sorted({0, s - 1})] + \
             [(23, 2, 1), (23, 8, 7)]


@pytest.mark.parametrize("log_m,stride,offset", _DECIMATED)
def test_ntt_decimated_exact(L, log_m, stride, offset):
    """pb200_fr_ntt_decimated: the 2^log_m-point transform of src[offset + stride * i], src exactly
    offset + stride * (m - 1) + 1 entries long; forward at every size, inverse up to 2^12"""
    m = 1 << log_m
    src = random_fr(offset + stride * (m - 1) + 1, 7 * log_m + stride + offset)
    sub = np.ascontiguousarray(src[offset::stride])
    assert sub.shape[0] == m
    d_src = to_dev(src)
    ctx = L.default_context().handle
    for inverse in ((False, True) if log_m <= 12 else (False,)):
        d_out = empty_dev(m)
        L.check(L.lib().pb200_fr_ntt_decimated(ctx, ptr(d_src), ptr(d_out), log_m, 1 if inverse else 0, stride, offset))
        out = to_host(d_out, L)
        if inverse:
            assert C.eval_coeffs(out, Z) == C.eval_lagrange(sub, Z)
        else:
            assert C.eval_lagrange(out, Z) == C.eval_coeffs(sub, Z)
    assert np.array_equal(to_host(d_src, L), src)  # the source is read only


# ------------------------------------------------------------------ coset transforms and barycentric evaluation
def _offsets(log_n):
    # every offset up to 2^20; 4n = 2^23 (three-pass) with the prover's coset and a random one, 4n = 2^24 with the
    # prover's coset
    return [1, COSET, OFFSET] if log_n <= 20 else [COSET, OFFSET] if log_n == 21 else [COSET]


@pytest.mark.parametrize("log_n", [0, 1, 9, 10, 11, 20, 21, 22])
def test_coset_extend_exact(L, log_n):
    """pb200_fr_coset_extend: n Lagrange values of P -> Q(y) = P(g y) on the 4n-th roots of unity, so
    eval_lagrange(out, z) == eval_lagrange(in, g z); the 4n transform crosses both pass boundaries"""
    n = 1 << log_n
    x = random_fr(n, 2000 + log_n)
    d_in = to_dev(x)
    for g in _offsets(log_n):
        d_out = empty_dev(4 * n)
        L.check(L.lib().pb200_fr_coset_extend(L.default_context().handle, ptr(d_in), ptr(d_out), log_n, fr_bytes(g)))
        out = to_host(d_out, L)
        assert C.eval_lagrange(out, Z) == C.eval_lagrange(x, g * Z % R), "offset %d" % g


@pytest.mark.parametrize("log_n", [0, 1, 2, 11, 12, 13, 22, 23, 24])
def test_coset_to_coeffs_exact(L, log_n):
    """pb200_fr_coset_to_coeffs: N values Q(y) = P(g y) on the N-th roots of unity -> the coefficients of P, so
    eval_coeffs(out, z) == eval_lagrange(in, z / g)"""
    n = 1 << log_n
    x = random_fr(n, 3000 + log_n)
    d_in = to_dev(x)
    for g in ([1, COSET, OFFSET] if log_n <= 13 else [OFFSET]):
        d_out = empty_dev(n)
        L.check(L.lib().pb200_fr_coset_to_coeffs(L.default_context().handle, ptr(d_in), ptr(d_out), log_n, fr_bytes(g)))
        out = to_host(d_out, L)
        assert C.eval_coeffs(out, Z) == C.eval_lagrange(x, Z * pow(g, -1, R) % R), "offset %d" % g


@pytest.mark.parametrize("log_n", [0, 1, 11, 12, 20, 23])
def test_barycentric_eval_exact(L, log_n):
    """pb200_fr_barycentric_eval against eval_lagrange at a random x and at x = 0; on the domain (x = w^k) it returns
    0 like the reference (inv(0) == 0, poly.py:181-195): against the Python oracle where it is cheap, else 0"""
    n = 1 << log_n
    x = random_fr(n, 4000 + log_n)
    d = to_dev(x)

    def bary(pt):
        out = ctypes.create_string_buffer(32)
        L.check(L.lib().pb200_fr_barycentric_eval(L.default_context().handle, ptr(d), log_n, fr_bytes(pt), out))
        return int.from_bytes(out.raw, "little")

    x_rand = random.Random(log_n).randrange(R)
    assert bary(x_rand) == C.eval_lagrange(x, x_rand)
    assert bary(0) == C.eval_lagrange(x, 0)
    w = O.root_of_unity(n)
    vals = [int.from_bytes(r.tobytes(), "little") for r in x] if n <= 4096 else None
    for k in sorted({0, 1, n // 2, n - 1}):
        on = pow(w, k, R)
        assert bary(on) == (O.barycentric_eval(vals, on) if vals is not None else 0) == 0, k
