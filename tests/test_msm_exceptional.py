"""GPU: commitments whose buckets add equal and opposite points -- the exceptional branches of the MSM's group law
(csrc/msm_bucket.cuh, csrc/curve.cuh) as compiled for sm_90a, checked exactly.

Random SRS points have unrelated discrete logs, so a bucket almost never holds P and P, or P and -P.  Here the SRS comes
from a degenerate tau, so its points collide by construction:
  tau = 1       every point is G: round 0 adds P + P (doublings), bucket sums are small multiples of G, so the
                reduction meets P == +-Q;
  tau = r - 1   G, -G, G, ...: P + (-P) in round 0, then identity slots carried through the later rounds;
  tau = w_4, w_8 (roots of unity) 4- and 8-cycles of points: both cases mixed;
  tau = 2, 2^c  the fixed-base table entry 2^(c w) P_i is the SRS point P_(i + w) (tau = 2^c), so in fixed-base mode,
                where all windows share one bucket set, one point reaches one bucket from different (i, w).
The check is that of tests/test_commit_exact.py: commit_coeffs(s) == [eval_coeffs(s, tau)]G (and the Lagrange form),
with its scalar patterns; on top, hand-built point lists through pb200_g1_msm_host, the point- and bucket-range shards
of one commitment joined on the host, and the refusal of the taus that would put the identity into an SRS.  The MSM
checks run twice: with the default XYZZ bucket accumulation, and in a child process with PB200_MSM_ACC=affine (read
once per process), whose batched affine additions classify equal x (P + P doubles, P + (-P) gives the identity)."""
import ctypes
import os
import random
import subprocess
import sys

import numpy as np
import pytest

from oracle import c_oracle as C
from oracle import plonk_oracle as O
from tests.test_commit_exact import PATTERNS, TAU, bucket_count, commit_coeffs, commit_lagrange, msm_generic, scalars
from tests.test_ntt_exact import ptr, to_dev

pytestmark = pytest.mark.gpu

R, Q = O.R_MOD, O.Q_MOD
W4, W8 = O.root_of_unity(4), O.root_of_unity(8)
DEGENERATE = {"one": lambda c: 1, "minus_one": lambda c: R - 1, "w4": lambda c: W4, "w8": lambda c: W8,
              "two": lambda c: 2, "two_pow_c": lambda c: 1 << c}


@pytest.fixture(scope="module")
def pb():
    import plonkathon_b200 as p
    return p


def sizes(k):
    return (1, 2, 3, 1 << k, (1 << k) + 3)


def eval_lagrange_any(v, tau):
    """value at tau of the polynomial with Lagrange values v on the n-th roots of unity, tau on the domain or off it"""
    n = v.shape[0]
    if pow(tau, n, R) != 1:
        return C.eval_lagrange(v, tau)
    w = O.root_of_unity(n)
    d = next(d for d in (1, 2, 4, 8, 16) if pow(tau, d, R) == 1)  # the order of tau, which divides n
    j = next(j for j in range(0, n, n // d) if pow(w, j, R) == tau)
    return int.from_bytes(v[j].tobytes(), "little")


def check_patterns(pb, setup, tau, c, ms, lagrange=True, tag=()):
    for m in ms:
        for k, name in enumerate(PATTERNS):
            s = scalars(name, m, c, 31 * c + 7 * m + k)
            assert commit_coeffs(pb, setup, s) == O.g1_multiply(O.G1, C.eval_coeffs(s, tau)), tag + (m, name)
            if lagrange and m & (m - 1) == 0:
                want = O.g1_multiply(O.G1, eval_lagrange_any(s, tau))
                assert commit_lagrange(pb, setup, s) == want, tag + (m, name, "lagrange")


# ------------------------------------------------------------------ fixed-base tables over degenerate SRSs
@pytest.mark.parametrize("tau_name", list(DEGENERATE))
@pytest.mark.parametrize("c", [4, 5, 8, 13, 16, 21])
def test_fixed_base_degenerate_tau(pb, monkeypatch, c, tau_name):
    """PB200_MSM_C_FIXED = c, SRS of 2^k + 3 points from a degenerate tau; every pattern at m = 1, 2, 3, 2^k, 2^k + 3
    (tau = 1 with all_equal at m > 2^12: one bucket of more than 4096 copies of G, the k_aff_tail rounds)"""
    monkeypatch.setenv("PB200_MSM_C_FIXED", str(c))
    tau = DEGENERATE[tau_name](c)
    k = 16 if c >= 16 else 12
    setup = pb.Setup.generate(tau, (1 << k) + 3)
    assert bucket_count(setup) == 1 << (c - 1)
    check_patterns(pb, setup, tau, c, sizes(k), tag=(c, tau_name))


@pytest.mark.parametrize("tau", [1, R - 1], ids=["one", "minus_one"])
def test_fixed_base_default_width_degenerate_tau(pb, monkeypatch, tau):
    """no environment: 2^21 + 6 points get c = 21; every point G (or +-G), every pattern at m = 1, 2, 3, 2^21 and
    2^21 + 6, the Lagrange form at 1, 2 and 2^21 points"""
    monkeypatch.delenv("PB200_MSM_C_FIXED", raising=False)
    n = (1 << 21) + 6
    setup = pb.Setup.generate(tau, n)
    assert bucket_count(setup) == 1 << 20
    check_patterns(pb, setup, tau, 21, (1, 2, 3, 1 << 21, n), tag=(tau,))


# ------------------------------------------------------------------ generic MSM over degenerate points
_generic = {}


def generic_setup(pb, tau_name, c):
    tau = DEGENERATE[tau_name](c)
    if tau not in _generic:
        _generic.clear()  # one SRS alive at a time
        n = (1 << 12) + 3
        setup = pb.Setup.generate(tau, n, precompute=False)
        _generic[tau] = (setup, setup.export_points_array(0, n))
    return tau, _generic[tau]


@pytest.mark.parametrize("tau_name", list(DEGENERATE))
@pytest.mark.parametrize("c", [4, 8, 13, 16])
def test_generic_degenerate_tau(pb, monkeypatch, c, tau_name):
    """PB200_MSM_C = c through pb200_g1_msm_host on the exported points and through an SRS built without the
    fixed-base table; every pattern at m = 1, 2, 3, 2^12, 2^12 + 3, and the Lagrange form"""
    monkeypatch.setenv("PB200_MSM_C", str(c))
    tau, (setup, pts) = generic_setup(pb, tau_name, c)
    assert bucket_count(setup) == 0
    for m in sizes(12):
        for k, name in enumerate(PATTERNS):
            s = scalars(name, m, c, 2000 + 31 * c + 7 * m + k)
            want = O.g1_multiply(O.G1, C.eval_coeffs(s, tau))
            assert msm_generic(pts, s) == want, (c, tau_name, m, name, "g1_msm")
            assert commit_coeffs(pb, setup, s) == want, (c, tau_name, m, name, "srs")
            if m & (m - 1) == 0:
                assert commit_lagrange(pb, setup, s) == O.g1_multiply(O.G1, eval_lagrange_any(s, tau)), (c, m, name)


# ------------------------------------------------------------------ hand-built point lists with known discrete logs
def _pool(pb):
    """{discrete log: affine point} for points exported from degenerate SRSs: G, -G, 2^i G, w_8^i G"""
    pool = {}
    for tau, n in ((1, 1), (R - 1, 2), (2, 16), (W8, 8)):
        setup = pb.Setup.generate(tau, n, precompute=False)
        raw = setup.export_points_array(0, n)
        for i in range(n):
            pool[pow(tau, i, R)] = raw[i].copy()
    assert pool[1].tobytes() == (1).to_bytes(32, "little") + (2).to_bytes(32, "little")  # G = (1, 2)
    assert pool[R - 1].tobytes() == (1).to_bytes(32, "little") + (Q - 2).to_bytes(32, "little")  # -G = (1, q - 2)
    return pool


def _lists(pool):
    rng = random.Random(77)
    keys = sorted(pool)
    lists = {
        "P_P_negP_P_2P": [1, 1, R - 1, 1, 2],
        "w8_P_P_negP_P_2P": [W8, W8, R - W8, W8, 2 * W8 % R],
        "run_of_one_point": [W8] * 300,
        "run_of_G_5000": [1] * 5000,
        "sums_to_identity": [1, 2, 4, R - 7],
        "P_negP_alternating": [W4, R - W4] * 150,
        "G_and_negG": [1, R - 1] * 64 + [1],
    }
    shuffled = [k for k in keys for _ in range(3)] + [(R - k) % R for k in keys]
    rng.shuffle(shuffled)
    lists["shuffled_pool_and_negatives"] = shuffled
    inter = []
    for k in keys:
        inter += [k, (R - k) % R, k, (2 * k) % R]
    lists["interleaved"] = inter
    return lists


def _point(pool, k):
    if k in pool:
        return pool[k]
    x, y = O.g1_multiply(O.G1, k)
    return np.frombuffer(x.to_bytes(32, "little") + y.to_bytes(32, "little"), dtype=np.uint8)


@pytest.mark.parametrize("c", [None, 4, 8])
def test_hand_built_point_lists(pb, monkeypatch, c):
    """pb200_g1_msm_host on lists of exported points with known discrete logs k_i (P, P, -P, P, 2P; runs of one
    point; lists summing to the identity; G = (1, 2) and -G = (1, q - 2) themselves): sum s_i P_i == (sum s_i k_i) G
    for every scalar pattern"""
    if c is None:
        monkeypatch.delenv("PB200_MSM_C", raising=False)
    else:
        monkeypatch.setenv("PB200_MSM_C", str(c))
    pool = _pool(pb)
    for lname, ks in _lists(pool).items():
        pts = np.stack([_point(pool, k) for k in ks])
        for j, name in enumerate(PATTERNS):
            s = scalars(name, len(ks), c or 8, 500 + 13 * j + len(ks))
            e = sum(int.from_bytes(s[i].tobytes(), "little") * k for i, k in enumerate(ks)) % R
            assert msm_generic(pts, s) == O.g1_multiply(O.G1, e), (c, lname, name)
        if lname == "sums_to_identity":
            assert msm_generic(pts, np.tile(scalars("all_equal", 1, 8, 3), (len(ks), 1))) is None


# ------------------------------------------------------------------ shards of one commitment, joined on the host
def _partial(pb, setup, d, first, count, lo, hi):
    from plonkathon_b200 import _lib
    out = ctypes.create_string_buffer(128)
    _lib.check(_lib.lib().pb200_srs_commit_partial(setup.ctx.handle, setup._srs, ptr(d), first, count, lo, hi, 0, out))
    return out.raw


@pytest.mark.parametrize("tau", [TAU, 1], ids=["random_tau", "one"])
def test_partial_commitments_join_to_full(pb, tau):
    """pb200_srs_commit_partial over the point ranges of parallel.shard_range and the bucket ranges of
    parallel.bucket_range (2, 3 and 4 parts, and both cuts at once), summed by pb200_g1_combine_partials_host,
    equal the full commitment"""
    from plonkathon_b200 import parallel
    n = (1 << 12) + 3
    setup = pb.Setup.generate(tau, n)
    nb = bucket_count(setup)
    for m in (n, 1 << 12, 5):
        for name in ("uniform", "all_equal", "r_minus_1", "half_zero"):
            s = scalars(name, m, 12, 900 + m)
            want = O.g1_multiply(O.G1, C.eval_coeffs(s, tau))
            assert commit_coeffs(pb, setup, s) == want
            d = to_dev(s)
            for world in (2, 3, 4):
                cuts = {
                    "points": [parallel.shard_range(m, r, world) + (0, nb) for r in range(world)],
                    "buckets": [(0, m) + parallel.bucket_range(nb, r, world) for r in range(world)],
                    "both": [parallel.shard_range(m, r, world) + parallel.bucket_range(nb, b, world)
                             for r in range(world) for b in range(world)],
                }
                for kind, parts in cuts.items():
                    raw = b"".join(_partial(pb, setup, d, *p) for p in parts)
                    xy, ident = parallel.combine_partials(raw, len(parts))
                    got = None if ident else (int.from_bytes(xy[:32], "little"), int.from_bytes(xy[32:], "little"))
                    assert got == want, (tau == 1, m, name, world, kind)


# ------------------------------------------------------------------ the batched-affine accumulation
@pytest.mark.skipif(os.environ.get("PB200_MSM_ACC") == "affine", reason="this process already runs the affine path")
def test_batched_affine_accumulation():
    """the MSM checks above again in a child process with PB200_MSM_ACC=affine (fixed-base c = 4, 13, 21 and the
    default width, generic c = 4, 13, every tau; the hand-built lists; the shards): round 0 pairs P with P and with -P
    (aff_classify_equal_x, the identity encoding x.v[7] == 0xffffffff), later rounds carry identity slots, and tau = 1
    with all_equal scalars runs the k_aff_tail rounds past PB_AFF_GRID_ROUNDS with a doubling at every step"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    me = os.path.abspath(__file__)
    ids = ["%s::test_fixed_base_degenerate_tau[%d-%s]" % (me, c, t) for c in (4, 13, 21) for t in DEGENERATE]
    ids += ["%s::test_generic_degenerate_tau[%d-%s]" % (me, c, t) for c in (4, 13) for t in DEGENERATE]
    ids += [me + "::test_fixed_base_default_width_degenerate_tau", me + "::test_hand_built_point_lists",
            me + "::test_partial_commitments_join_to_full"]
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider"] + ids,
                       cwd=root, env=dict(os.environ, PB200_MSM_ACC="affine"), capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
    assert " passed" in r.stdout and "skipped" not in r.stdout, r.stdout[-2000:]


# ------------------------------------------------------------------ taus that would put the identity into an SRS
def _small_proof_verifies(pb):
    from plonkathon_b200 import synthetic as syn
    log_n = 5
    n = 1 << log_n
    circ = syn.build_circuit(log_n, seed=5, n_public=1)
    pk, A, B, Cw, public = syn.circuit_arrays(circ)
    setup = pb.Setup.generate(TAU, n + 6)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, Cw, public)
    return setup.verification_key_arrays(n, pk).verify_proof(n, pb.Proof.from_bytes(raw), [int(x) for x in public])


def test_tau_zero_refused(pb):
    """tau = 0 mod r: Setup.generate raises ValueError, pb200_srs_generate returns an error that names the condition,
    and the context still commits and proves"""
    from plonkathon_b200 import _lib
    for tau in (0, R, 5 * R):
        with pytest.raises(ValueError, match="tau == 0"):
            pb.Setup.generate(tau, 64)
    h = ctypes.c_void_p()
    ctx = _lib.default_context()
    for precompute in (0, 1):
        assert _lib.lib().pb200_srs_generate(ctx.handle, bytes(32), 64, precompute, ctypes.byref(h)) != 0
        assert "tau == 0" in _lib.lib().pb200_last_error().decode()
        assert not h.value
    setup = pb.Setup.generate(1, 64)
    s = scalars("uniform", 64, 8, 1)
    assert commit_coeffs(pb, setup, s) == O.g1_multiply(O.G1, C.eval_coeffs(s, 1))
    assert _small_proof_verifies(pb)


@pytest.mark.parametrize("log_n", [0, 1, 3, 10])
def test_lagrange_tau_on_domain_refused(pb, log_n):
    """tau^n = 1 (tau = w_n^k): enable_lagrange(n) raises ValueError, pb200_srs_generate_lagrange returns an error
    that names the condition; a tau of order 2n (just off the domain) is accepted and commits exactly"""
    from plonkathon_b200 import _lib
    n = 1 << log_n
    w = O.root_of_unity(n)
    ctx = _lib.default_context()
    for k in sorted({0, 1, n // 2, n - 1}):
        tau = pow(w, k, R)
        setup = pb.Setup.generate(tau, n, precompute=False)  # the monomial SRS is fine
        with pytest.raises(ValueError, match=r"tau\^n == 1"):
            setup.enable_lagrange(n)
        h = ctypes.c_void_p()
        assert _lib.lib().pb200_srs_generate_lagrange(ctx.handle, tau.to_bytes(32, "little"), n, 0, ctypes.byref(h)) != 0
        assert "tau^n == 1" in _lib.lib().pb200_last_error().decode()
        assert not h.value
    tau = O.root_of_unity(2 * n)
    setup = pb.Setup.generate(tau, n)
    assert setup.enable_lagrange(n)
    v = scalars("uniform", n, 8, 40 + log_n)
    d = np.ascontiguousarray(v)
    out, ident = ctypes.create_string_buffer(64), ctypes.c_int(-1)
    _lib.check(_lib.lib().pb200_srs_commit_coeffs_host(ctx.handle, setup._lagrange[n], d.ctypes.data_as(ctypes.c_void_p),
                                                       n, out, ctypes.byref(ident)))
    got = None if ident.value else (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little"))
    assert got == O.g1_multiply(O.G1, C.eval_lagrange(v, tau))
    assert _small_proof_verifies(pb)
