"""GPU: KZG commitments (the G1 MSM) checked exactly at every window width the MSM can run with.

Against the structured SRS [tau^i]G of a known tau, commit_coeffs(s) == [eval_coeffs(s, tau)]G and
commit_lagrange(v) == [eval_lagrange(v, tau)]G: one O(m) evaluation by the C restatement (oracle/c/plonk_oracle.c)
and one host scalar multiplication per commitment.  The window width c changes the digit slicing, the bucket counts,
the segment length and the reduction groups, so every width is run with scalar patterns that stress the signed
digits (r - 1 carries out of every window; digits of exactly 2^(c-1) sit on the carry boundary) and the heavy-bucket
path (every scalar equal: one bucket per window holds every entry).  Fixed-base tables take c = 4..21
(PB200_MSM_C_FIXED, read when an SRS is built), generic MSMs c = 4..16 (PB200_MSM_C, read on every call); every SRS
of more than 2^20 points gets c = 21, checked here at 2^21 + 6 (a zero-knowledge prover's SRS) and 2^22 points."""
import ctypes
import random

import numpy as np
import pytest

from oracle import c_oracle as C
from oracle import plonk_oracle as O

pytestmark = pytest.mark.gpu

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
PATTERNS = ("uniform", "r_minus_1", "all_equal", "digit_half", "zero", "last_only", "half_zero")


@pytest.fixture(scope="module")
def pb():
    import plonkathon_b200 as p
    return p


def row(x):
    return np.frombuffer((int(x) % R).to_bytes(32, "little"), dtype=np.uint32)


def digit_half_scalar(c):
    """every c-bit digit below bit 253 equal to 2^(c-1): the signed-digit carry boundary in every window"""
    return sum(1 << (c * w + c - 1) for w in range(256) if c * w + c - 1 < 253)


def scalars(name, m, c, seed):
    rng = np.random.default_rng(seed)
    if name == "uniform":  # all 254 bits in use (bits 252 and 253 feed the top window), every value below r
        a = rng.integers(0, 1 << 32, size=(m, 8), dtype=np.uint32)
        a[:, 7] &= 0x3FFFFFFF
        a[a[:, 7] >= 0x30644E72, 7] = 0x30644E71  # r's top limb is 0x30644E72
        return a
    if name == "r_minus_1":
        return np.tile(row(R - 1), (m, 1))
    if name == "all_equal":
        return np.tile(row(random.Random(seed).randrange(1, R)), (m, 1))
    if name == "digit_half":
        return np.tile(row(digit_half_scalar(c)), (m, 1))
    a = scalars("uniform", m, c, seed)
    if name == "zero":
        a[:] = 0
    elif name == "last_only":
        a[:m - 1] = 0
    elif name == "half_zero":
        a[::2] = 0
    return a


def point(out, ident):
    return None if ident.value else (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little"))


def commit_coeffs(pb, setup, s):
    from plonkathon_b200 import _lib
    out, ident = ctypes.create_string_buffer(64), ctypes.c_int(-1)
    _lib.check(_lib.lib().pb200_srs_commit_coeffs_host(setup.ctx.handle, setup._srs, s.ctypes.data_as(ctypes.c_void_p),
                                                       s.shape[0], out, ctypes.byref(ident)))
    return point(out, ident)


def commit_lagrange(pb, setup, v):
    from plonkathon_b200 import _lib
    out, ident = ctypes.create_string_buffer(64), ctypes.c_int(-1)
    _lib.check(_lib.lib().pb200_srs_commit_lagrange_host(setup.ctx.handle, setup._srs, v.ctypes.data_as(ctypes.c_void_p),
                                                         v.shape[0].bit_length() - 1, out, ctypes.byref(ident)))
    return point(out, ident)


def msm_generic(pts, s):
    from plonkathon_b200 import _lib
    out, ident = ctypes.create_string_buffer(64), ctypes.c_int(-1)
    m = s.shape[0]
    _lib.check(_lib.lib().pb200_g1_msm_host(_lib.default_context().handle, pts[:m].ctypes.data_as(ctypes.c_void_p),
                                            s.ctypes.data_as(ctypes.c_void_p), m, out, ctypes.byref(ident)))
    return point(out, ident)


def expect_coeffs(s):
    return O.g1_multiply(O.G1, C.eval_coeffs(s, TAU))


def bucket_count(setup):
    from plonkathon_b200 import _lib
    out = ctypes.c_uint(0)
    _lib.check(_lib.lib().pb200_srs_bucket_count(setup._srs, ctypes.byref(out)))
    return out.value


def _check_all_patterns(pb, setup, c, sizes, lagrange=True):
    for m in sizes:
        for k, name in enumerate(PATTERNS):
            s = scalars(name, m, c, 100 * c + 7 * m + k)
            got = commit_coeffs(pb, setup, s)
            assert got == expect_coeffs(s), (c, m, name)
            if name == "zero":
                assert got is None  # is_identity == 1
            if lagrange and m & (m - 1) == 0:
                assert commit_lagrange(pb, setup, s) == O.g1_multiply(O.G1, C.eval_lagrange(s, TAU)), (c, m, name, "lag")


# ------------------------------------------------------------------ fixed-base table, every width
@pytest.mark.parametrize("c", range(4, 22))
def test_fixed_base_every_window_exact(pb, monkeypatch, c):
    """PB200_MSM_C_FIXED = c for a small SRS (2^12 + 3 points, 2^16 + 3 from c = 16): the table has
    ceil(256 / c) windows of 2^(c-1) signed buckets; m = 1, 2^k and 2^k + 3 scalars of every pattern"""
    monkeypatch.setenv("PB200_MSM_C_FIXED", str(c))
    k = 16 if c >= 16 else 12
    setup = pb.Setup.generate(TAU, (1 << k) + 3)
    assert bucket_count(setup) == 1 << (c - 1)
    _check_all_patterns(pb, setup, c, (1, 1 << k, (1 << k) + 3))


# ------------------------------------------------------------------ generic MSM, every width
@pytest.fixture(scope="module")
def generic_setup(pb):
    n = (1 << 12) + 3
    setup = pb.Setup.generate(TAU, n, precompute=False)
    return setup, setup.export_points_array(0, n)


@pytest.mark.parametrize("c", range(4, 17))
def test_generic_every_window_exact(pb, generic_setup, monkeypatch, c):
    """PB200_MSM_C = c through pb200_g1_msm (SRS points exported to the host) and through an SRS built without the
    fixed-base table; every pattern at m = 1, 2^12, 2^12 + 3"""
    monkeypatch.setenv("PB200_MSM_C", str(c))
    setup, pts = generic_setup
    assert bucket_count(setup) == 0  # no table: the window is chosen per call
    for m in (1, 1 << 12, (1 << 12) + 3):
        for k, name in enumerate(PATTERNS):
            s = scalars(name, m, c, 1000 + 100 * c + 7 * m + k)
            want = expect_coeffs(s)
            assert msm_generic(pts, s) == want, (c, m, name, "g1_msm")
            assert commit_coeffs(pb, setup, s) == want, (c, m, name, "srs")
            if name == "zero":
                assert want is None


# ------------------------------------------------------------------ the default width at full size: c = 21
@pytest.mark.parametrize("log_n,extra", [(21, 6), (22, 0)])
def test_fixed_base_default_width_full_size(pb, monkeypatch, log_n, extra):
    """no environment: an SRS of more than 2^20 points gets c = 21 (13 windows, the top one holding bits 252-253,
    so four heavy buckets take every entry between them); every pattern at m = 1, 2^log_n and the SRS size"""
    monkeypatch.delenv("PB200_MSM_C_FIXED", raising=False)
    n = (1 << log_n) + extra
    setup = pb.Setup.generate(TAU, n)
    assert bucket_count(setup) == 1 << 20
    sizes = (1, 1 << log_n) + ((n,) if extra else ())
    for m in sizes:
        for k, name in enumerate(PATTERNS):
            s = scalars(name, m, 21, 5000 + 7 * m + k)
            assert commit_coeffs(pb, setup, s) == expect_coeffs(s), (m, name)
    v = scalars("uniform", 1 << log_n, 21, 77)
    assert commit_lagrange(pb, setup, v) == O.g1_multiply(O.G1, C.eval_lagrange(v, TAU))


def test_zero_knowledge_proof_2p21_gates_verifies(pb):
    """a zero-knowledge proof at 2^21 gates: its commitments have n + 3 coefficients against an SRS of n + 6 powers
    (c = 21, lengths that are not powers of two, the batched commitments of 2 and 3 vectors); the verifier accepts it
    and rejects a changed evaluation"""
    import torch
    if torch.cuda.get_device_properties(0).total_memory < 60 * 2 ** 30:
        pytest.skip("needs ~30 GB of HBM")
    from plonkathon_b200 import synthetic as syn
    log_n = 21
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=21, n_public=2)
    pk, A, B, Cw, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n + 6)
    assert bucket_count(setup) == 1 << 20
    prover = pb.Prover.from_arrays(setup, n, pk)
    prover.set_zk(True, [random.Random(21).randrange(R) for _ in range(11)])
    raw = prover.prove_arrays(A, B, Cw, public)
    vk = setup.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), pub)
    k = 32 * 14  # a_eval
    bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not vk.verify_proof(n, pb.Proof.from_bytes(bad), pub)
