"""GPU parity tests (run on an H100): the CUDA path, called through the C ABI / the drop-in
Python surface, against the oracle (oracle/plonk_oracle.py) on the same seeded inputs, against the
committed golden fixtures, and -- at BASELINE.json's full sizes -- through size-independent
properties.  Bit-exact everywhere (integer field work)."""
import ctypes
import random

import numpy as np
import pytest

from oracle import plonk_oracle as O
from tests.golden_io import PTAU_HEAD, ints, load_circuit, load_json, pt

pytestmark = pytest.mark.gpu

R = O.R_MOD


@pytest.fixture(scope="module")
def pb():
    import plonkathon_b200 as p
    return p


@pytest.fixture(scope="module")
def setup(pb):
    return pb.Setup.from_file(PTAU_HEAD)


def S(pb, ints_):
    return [pb.Scalar(v) for v in ints_]


def vals(poly):
    return [v.n for v in poly.values]


# ------------------------------------------------------------------ NTT
def test_fft_golden_vectors(pb):
    for c in load_json("fft_vectors.json")["cases"]:
        v = ints(c["input"])
        assert vals(pb.Polynomial(S(pb, v), pb.Basis.MONOMIAL).fft()) == ints(c["fft"]), c["n"]
        L = pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE)
        assert vals(L.ifft()) == ints(c["ifft"]), c["n"]
        if "offset" in c:
            off = pb.Scalar(int(c["offset"]))
            assert vals(L.to_coset_extended_lagrange(off)) == ints(c["coset_ext"])
            assert vals(L.coset_extended_lagrange_to_coeffs(off)) == ints(c["coset_to_coeffs"])
            assert L.barycentric_eval(pb.Scalar(int(c["x"]))) == int(c["bary"])
            assert L.barycentric_eval(pb.Scalar(int(c["x_root"]))) == int(c["bary_root"])


def test_fft_basis_assertions(pb):
    p = pb.Polynomial(S(pb, [1, 2]), pb.Basis.LAGRANGE)
    with pytest.raises(AssertionError):
        p.fft()
    with pytest.raises(AssertionError):
        pb.Polynomial(S(pb, [1, 2]), pb.Basis.MONOMIAL).ifft()


@pytest.mark.parametrize("logn", [11, 12, 13, 14, 16])
def test_fft_vs_oracle_multi_pass(pb, logn):
    rng = random.Random(logn)
    v = [rng.randrange(R) for _ in range(1 << logn)]
    assert vals(pb.Polynomial(S(pb, v), pb.Basis.MONOMIAL).fft()) == O.fft(v)
    assert vals(pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE).ifft()) == O.ifft(v)


def _raw_ntt(pb, arr, logn, inverse):
    from plonkathon_b200 import _lib
    out = np.empty_like(arr)
    _lib.check(_lib.lib().pb200_fr_ntt_host(
        _lib.default_context().handle, arr.ctypes.data_as(ctypes.c_void_p),
        out.ctypes.data_as(ctypes.c_void_p), logn, inverse))
    return out


def _random_fr(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 1 << 32, size=(n, 8), dtype=np.uint64).astype(np.uint32)
    a[:, 7] &= 0x0FFFFFFF  # < 2^252 < r: canonical
    return a


@pytest.mark.parametrize("logn", [20, 21, 22])
def test_ntt_full_size_properties(pb, logn):
    """2^20 .. 2^22 (two-pass: ntt.cu runs one pass up to 2^11, two up to 2^22, three from 2^23; the three-pass sizes
    are checked in tests/test_ntt_exact.py): inverse(forward(x)) == x, linearity against a sparse
    input whose transform is known in closed form, and a strided sample against the oracle's
    direct evaluation."""
    n = 1 << logn
    x = _random_fr(n, logn)
    y = _raw_ntt(pb, x, logn, 0)
    back = _raw_ntt(pb, y, logn, 1)
    assert np.array_equal(back, x)
    # direct evaluation at a few output indices: X[k] = sum_j x[j] w^(jk) computed with Python ints
    xs = [int.from_bytes(x[j].tobytes(), "little") for j in range(n)] if logn == 20 else None
    if xs is not None:
        w = O.root_of_unity(n)
        for k in (0, 1, n // 2 + 3, n - 1):
            wk = pow(w, k, R)
            acc, cur = 0, 1
            for j in range(n):
                acc += xs[j] * cur
                cur = cur * wk % R
            assert int.from_bytes(y[k].tobytes(), "little") == acc % R, k
    # delta at position p: transform is w^(p*k)
    d = np.zeros((n, 8), dtype=np.uint32)
    p = 12345 % n
    d[p, 0] = 1
    yd = _raw_ntt(pb, d, logn, 0)
    w = O.root_of_unity(n)
    for k in (0, 1, 2, n // 3, n - 1):
        assert int.from_bytes(yd[k].tobytes(), "little") == pow(w, p * k, R)


# ------------------------------------------------------------------ MSM
def test_lincomb_golden_vectors(pb):
    for c in load_json("lincomb_vectors.json")["cases"]:
        pairs = [(None if p is None else (pb.FQ(int(p[0])), pb.FQ(int(p[1]))), int(s))
                 for p, s in zip(c["points"], c["scalars"])]
        got = pb.ec_lincomb(pairs)
        exp = pt(c["result"])
        assert (got is None and exp is None) or (got[0].n, got[1].n) == exp, c["name"]


def test_lincomb_empty_raises(pb):
    with pytest.raises(ValueError):
        pb.ec_lincomb([])


@pytest.mark.parametrize("n", [1, 3, 257, 1024])
def test_lincomb_vs_oracle_random(pb, n):
    rng = random.Random(n)
    osetup = O.Setup.from_file(PTAU_HEAD)
    pts = osetup.powers_of_x[:n]
    sc = [rng.randrange(R) for _ in range(n)]
    got = pb.ec_lincomb([((pb.FQ(p[0]), pb.FQ(p[1])), s) for p, s in zip(pts, sc)])
    exp = O.ec_lincomb_naive(list(zip(pts, sc))) if n <= 3 else O.ec_lincomb(list(zip(pts, sc)))
    assert (got[0].n, got[1].n) == exp


def test_commit_kat_and_vkeys(pb, setup):
    """test.py:14-34 commitment KAT, and the three snarkjs verification keys (test.py:37-100)."""
    g = load_json("circuits.json")
    c = setup.commit(pb.Polynomial(S(pb, ints(g["commit_kat"]["lagrange"])), pb.Basis.LAGRANGE))
    assert c == (16120260411117808045030798560855586501988622612038310041007562782458075125622,
                 3125847109934958347271782137825877642397632921923926105820408033549219695465)
    for name in ("basic", "ab_plus_a", "one_public"):
        entry, arr = load_circuit(name)
        for key, col in (("Qm", "QM"), ("Ql", "QL"), ("Qr", "QR"), ("Qo", "QO"), ("Qc", "QC"),
                         ("S1", "S1"), ("S2", "S2"), ("S3", "S3")):
            got = setup.commit(pb.Polynomial(S(pb, arr[col]), pb.Basis.LAGRANGE))
            exp = pt(entry["vk"][key])
            assert (got is None and exp is None) or (got[0].n, got[1].n) == exp, (name, key)


def test_commit_generic_equals_fixed_base(pb):
    """the two MSM modes (generic windows vs precomputed fixed-base table) agree"""
    s1 = pb.Setup.from_file(PTAU_HEAD, precompute=True)
    s2 = pb.Setup.from_file(PTAU_HEAD, precompute=False)
    rng = random.Random(3)
    for n in (8, 512, 2048):
        p = pb.Polynomial(S(pb, [rng.randrange(R) for _ in range(n)]), pb.Basis.LAGRANGE)
        a, b = s1.commit(p), s2.commit(p)
        assert (a[0].n, a[1].n) == (b[0].n, b[1].n)
    osetup = O.Setup.from_file(PTAU_HEAD)
    v = [rng.randrange(R) for _ in range(2048)]
    got = s1.commit(pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE))
    assert (got[0].n, got[1].n) == osetup.commit(v)


def test_msm_2p20_repeated_bases(pb):
    """KZG-size MSM (2^20 terms) with an exactly-known answer: the 2048 SRS points tiled 512x, so
    sum_i s_i P_(i mod 2048) == sum_j (sum_(i = j mod 2048) s_i) P_j, which the oracle evaluates
    as a 2048-term ec_lincomb.  Also exercises repeated base points inside one MSM."""
    from plonkathon_b200 import _lib
    osetup = O.Setup.from_file(PTAU_HEAD)
    base = np.frombuffer(b"".join(p[0].to_bytes(32, "little") + p[1].to_bytes(32, "little")
                                  for p in osetup.powers_of_x), dtype=np.uint8).reshape(2048, 64)
    n = 1 << 20
    pts = np.ascontiguousarray(np.tile(base, (n // 2048, 1)))
    sc = _random_fr(n, 99)
    out = ctypes.create_string_buffer(64)
    ident = ctypes.c_int(0)
    _lib.check(_lib.lib().pb200_g1_msm_host(
        _lib.default_context().handle, pts.ctypes.data_as(ctypes.c_void_p),
        sc.ctypes.data_as(ctypes.c_void_p), n, out, ctypes.byref(ident)))
    # fold the scalars per base point with exact integer arithmetic
    limbs = sc.astype(object)
    folded = [0] * 2048
    rows = limbs.reshape(n // 2048, 2048, 8)
    for k in range(8):
        col = rows[:, :, k].sum(axis=0)
        for j in range(2048):
            folded[j] += int(col[j]) << (32 * k)
    exp = O.ec_lincomb([(osetup.powers_of_x[j], folded[j] % R) for j in range(2048)])
    got = (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little"))
    assert ident.value == 0 and got == exp


# ------------------------------------------------------------------ transcript (host code, in the .so)
def test_transcript_vectors(pb):
    g = load_json("circuits.json")
    t = pb.Transcript(b"test protocol")
    t.append_message(b"some label", b"some data")
    assert t.challenge_bytes(b"challenge", 32).hex() == g["merlin_vector"]
    tr = pb.Transcript(b"plonk")
    tr.append_point(b"a_1", (pb.FQ(1), pb.FQ(2)))
    tr.append_scalar(b"a_eval", pb.Scalar(12345))
    assert tr.get_and_append_challenge(b"beta") == int(g["transcript"]["beta"])
    assert tr.get_and_append_challenge(b"gamma") == int(g["transcript"]["gamma"])


# ------------------------------------------------------------------ full proofs
def _pk(arr):
    return {k: arr[k] for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")}


@pytest.mark.parametrize("name", ["prover_test", "factorization", "poseidon"])
def test_prove_golden_circuits(pb, setup, name):
    """Bit-identical 768-byte proofs: prover_test == the reference's test/proof.pickle; factorization and
    mini-Poseidon (test.py:171-259) == proofs the reference's own verifier accepted at fixture time."""
    import hashlib
    entry, arr = load_circuit(name)
    prover = pb.Prover.from_arrays(setup, entry["n"], _pk(arr))
    raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"]
    proof = pb.Proof.from_bytes(raw).flatten()
    for k, v in entry["proof"].items():
        got = proof[k]
        assert ((got[0].n, got[1].n) == pt(v)) if isinstance(v, list) else (got.n == int(v)), k
    # second proof with the same prover object (state reuse) is identical
    assert prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"])) == raw


def test_prove_through_reference_surface(pb, setup):
    """Prover(setup, program).prove(witness) with a Program-shaped object (test.py:136-145): the round-by-round
    path with the Python Transcript gives the same proof as test/proof.pickle."""
    from collections import namedtuple
    entry, arr = load_circuit("prover_test")
    W = namedtuple("GateWires", "L R O")
    P = namedtuple("Poly", "values")
    PK = namedtuple("PK", "group_order QM QL QR QO QC S1 S2 S3")

    class Program:  # ["e public", "c <== a * b", "e <== c * d"], group order 8
        group_order = 8

        def common_preprocessed_input(self):
            return PK(8, *[P([pb.Scalar(v) for v in arr[k]]) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")])

        def wires(self):
            return [W("e", None, None), W("a", "b", "c"), W("c", "d", "e")]

        def get_public_assignments(self):
            return ["e"]

    witness = {"a": 3, "b": 4, "c": 12, "d": 5, "e": 60}
    proof = pb.Prover(setup, Program()).prove(witness)
    assert witness[None] == 0  # prover.py:94-95 mutates the witness
    import hashlib
    assert hashlib.sha256(proof.to_bytes()).hexdigest() == \
        "4550f3296053d1b17252c41453680871b280af947381d270241c2957c730eeb1"


def test_prove_rejects_bad_witness(pb, setup):
    entry, arr = load_circuit("factorization")
    prover = pb.Prover.from_arrays(setup, entry["n"], _pk(arr))
    bad = list(arr["C"])
    bad[15] = (bad[15] + 1) % R
    with pytest.raises(AssertionError):  # prover.py:108-116
        prover.prove_arrays(arr["A"], arr["B"], bad, ints(entry["public"]))


# ------------------------------------------------------------------ synthetic SRS + circuits
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF


def test_srs_generate_matches_oracle(pb):
    s = pb.Setup.generate(TAU, 300, precompute=False)
    got = [(p[0].n, p[1].n) for p in s.export_points(0, 300)]
    cur = O.G1
    for i in range(300):
        assert got[i] == cur, i
        cur = O.g1_multiply(cur, TAU)


@pytest.mark.parametrize("log_n,fill", [(4, 1.0), (7, 0.9)])
def test_prove_synthetic_vs_oracle(pb, log_n, fill):
    """synthetic circuit family used by bench.py, small instance: GPU proof bytes == oracle proof bytes"""
    from plonkathon_b200 import synthetic as syn
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=log_n, n_public=2, fill=fill)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, C, public)
    S1, S2, S3 = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    opk = O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3)
    osetup = O.Setup([(p[0].n, p[1].n) for p in setup.powers_of_x], None)
    a, b, cc = c.wires_values()
    assert raw == O.proof_bytes(O.Prover(osetup, opk).prove(a, b, cc, c.public_values()))


def test_prove_2p20_gates_verifies(pb):
    """BASELINE.json's headline size: a 2^20-gate synthetic circuit.  The reference cannot produce a proof
    at this size (5 h of Python; SRS file holds 2^11 powers); parity is established byte for byte against the
    golden proof of the oracle prover run over the C restatement, and end to end by the
    reference's verification equation (TESTING_verifier_DO_NOT_OPEN.py:39-163) evaluated by the oracle with
    the known tau of the structured SRS, plus independent CPU evaluation of two verification-key
    commitments, plus determinism (two runs, host-buffer and device-buffer paths agree in bench.py)."""
    from plonkathon_b200 import synthetic as syn
    log_n = 20
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=7, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk)
    raw = prover.prove_arrays(A, B, C, public)
    assert prover.prove_arrays(A, B, C, public) == raw
    # byte for byte against the oracle's proof of the same circuit (tests/golden/make_proof_2p20.py: the oracle prover
    # over the C restatement of fft / ec_lincomb, ~20 CPU-minutes, committed as a fixture)
    import json
    import os
    from tests.golden_io import GOLDEN
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    assert rec["log_n"] == log_n and rec["seed"] == 7 and [int(x) for x in rec["public"]] == [int(x) for x in public]
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden proof at 2^20 gates"
    proof = O.proof_from_bytes(raw)
    for k in ("a_1", "z_1", "t_hi_1", "W_zw_1"):
        assert O.g1_is_on_curve(proof[k])

    def commit(col):
        import ctypes
        from plonkathon_b200 import _lib
        out = ctypes.create_string_buffer(64)
        ident = ctypes.c_int()
        _lib.check(_lib.lib().pb200_srs_commit_lagrange_host(
            setup.ctx.handle, setup._srs, pk[col].ctypes.data_as(ctypes.c_void_p), log_n, out, ctypes.byref(ident)))
        return None if ident.value else (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little"))

    vk = {k: commit(col) for k, col in (("Qm", "QM"), ("Ql", "QL"), ("Qr", "QR"), ("Qo", "QO"), ("Qc", "QC"),
                                        ("S1", "S1"), ("S2", "S2"), ("S3", "S3"))}
    # two of the eight commitments re-derived on the CPU: [f(tau)] G with f evaluated from its Lagrange values
    S1, _, _ = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    assert vk["S1"] == O.g1_multiply(O.G1, O.eval_lagrange_at(S1, TAU))
    assert vk["Qm"] == O.g1_multiply(O.G1, O.eval_lagrange_at(c.QM, TAU))
    assert O.verify_proof_trapdoor(n, vk, proof, public, TAU)
    bad = dict(proof)
    bad["z_shifted_eval"] = (bad["z_shifted_eval"] + 1) % R
    assert not O.verify_proof_trapdoor(n, vk, bad, public, TAU)
    # and by the product's own verifier: GPU linear combinations + the BN254 pairing against X2 = [tau]_2
    pvk = setup.verification_key_arrays(n, pk)
    assert all((getattr(pvk, k)[0].n, getattr(pvk, k)[1].n) == vk[k] for k in vk)
    pub_ints = [int(x) for x in public]
    assert pvk.verify_proof(n, pb.Proof.from_bytes(raw), pub_ints)
    assert pvk.verify_proof_unoptimized(n, pb.Proof.from_bytes(raw), pub_ints)
    k = 32 * 19
    raw_bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not pvk.verify_proof(n, pb.Proof.from_bytes(raw_bad), pub_ints)
    assert not pvk.verify_proof(n, pb.Proof.from_bytes(raw), [pub_ints[0] + 1] + pub_ints[1:])


def test_prove_many_public_inputs_dense_path(pb):
    """more than 8 public inputs take the generic (interpolated PI) path; same bytes as the oracle"""
    from plonkathon_b200 import synthetic as syn
    log_n = 6
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=3, n_public=11)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, C, public)
    S1, S2, S3 = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    opk = O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3)
    osetup = O.Setup([(p[0].n, p[1].n) for p in setup.powers_of_x], None)
    a, b, cc = c.wires_values()
    assert raw == O.proof_bytes(O.Prover(osetup, opk).prove(a, b, cc, c.public_values()))


@pytest.mark.parametrize("log_n,n_public", [(12, 12), (13, 2)])
def test_prove_mid_size_vs_oracle(pb, log_n, n_public):
    """mid-size differential against the oracle prover (its fft / ec_lincomb answered by the C restatement,
    oracle/fast.py -- byte-identical to the pure-Python oracle, tests/test_oracle_fast.py): the two-pass NTT regime
    (4n = 2^14, 2^15: tiles of several columns), and more than 8 public inputs through the interpolated-PI branch at a size where it
    crosses tile boundaries"""
    from oracle import fast as F
    from plonkathon_b200 import synthetic as syn
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=40 + log_n, n_public=n_public)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, C, public)
    S1, S2, S3 = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    opk = O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3)
    a, b, cc = c.wires_values()
    assert raw == O.proof_bytes(F.prove(F.Setup(TAU, n), opk, a, b, cc, c.public_values()))


def test_verification_key_object(pb, setup):
    """Setup.verification_key(pk) (setup.py:75-77) with a CommonPreprocessedInput-shaped object"""
    from collections import namedtuple
    entry, arr = load_circuit("one_public")
    P = namedtuple("Poly", "values basis")
    PK = namedtuple("PK", "group_order QM QL QR QO QC S1 S2 S3")
    pk = PK(8, *[pb.Polynomial(S(pb, arr[k]), pb.Basis.LAGRANGE) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")])
    vk = setup.verification_key(pk)
    for key in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
        got, exp = getattr(vk, key), pt(entry["vk"][key])
        assert (got is None and exp is None) or (got[0].n, got[1].n) == exp, key
    assert vk.w == int(entry["vk"]["w"]) and vk.group_order == 8
    assert (tuple(vk.X_2[0]), tuple(vk.X_2[1])) == tuple(tuple(int(c) for c in row) for row in entry["vk"]["X_2"])


def test_msm_skewed_scalars_2p18(pb):
    """witness-like scalar distribution (half zeros, a quarter ones, small constants, the rest uniform) through
    the fixed-base commit path: exact answer by folding per base point, and no load-imbalance blow-up"""
    import time
    from plonkathon_b200 import _lib
    n = 1 << 18
    setup = pb.Setup.generate(TAU, n)
    rng = np.random.default_rng(5)
    sc = _random_fr(n, 17)
    kind = rng.integers(0, 8, size=n)
    sc[kind < 4] = 0
    ones = (kind == 4) | (kind == 5)
    sc[ones] = 0
    sc[ones, 0] = 1
    small = kind == 6
    sc[small] = 0
    sc[small, 0] = rng.integers(2, 1000, size=int(small.sum()))
    out = ctypes.create_string_buffer(64)
    ident = ctypes.c_int(0)
    dev = __import__("torch").from_numpy(sc.view(np.int32)).cuda()
    t0 = time.time()
    _lib.check(_lib.lib().pb200_srs_commit_coeffs(setup.ctx.handle, setup._srs, ctypes.c_void_p(dev.data_ptr()), n, 0,
                                                  out, ctypes.byref(ident)))
    dt = time.time() - t0
    # expected: sum_i s_i tau^i * G
    acc, cur = 0, 1
    sc_int = [int.from_bytes(sc[i].tobytes(), "little") for i in range(n)]
    for s_i in sc_int:
        if s_i:
            acc += s_i * cur
        cur = cur * TAU % R
    exp = O.g1_multiply(O.G1, acc % R)
    got = (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little"))
    assert got == exp
    assert dt < 0.5, "skewed MSM took %.3f s" % dt


def test_error_behaviour_matches_reference(pb, setup):
    """errors surface as the reference's exception types at the boundary"""
    big = pb.Polynomial(S(pb, list(range(4096))), pb.Basis.LAGRANGE)
    with pytest.raises(Exception, match="Not enough powers"):  # SRS holds 2^11 powers (setup.py:27)
        setup.commit(big)
    with pytest.raises(AssertionError):  # setup.py:67 asserts the LAGRANGE basis
        setup.commit(pb.Polynomial(S(pb, [1, 2]), pb.Basis.MONOMIAL))
    with pytest.raises(AssertionError):  # poly.py:15 isinstance check
        pb.Polynomial([1, 2], pb.Basis.LAGRANGE)
    with pytest.raises(AssertionError):  # power-of-two length
        pb.Polynomial(S(pb, [1, 2, 3]), pb.Basis.MONOMIAL).fft()
    with pytest.raises(AssertionError):  # poly.py:157 basis assert
        pb.Polynomial(S(pb, [1, 2]), pb.Basis.MONOMIAL).to_coset_extended_lagrange(pb.Scalar(3))
    # scalars >= r and negative ints are reduced like curve.py:41
    g = (pb.FQ(1), pb.FQ(2))
    a = pb.ec_lincomb([(g, -1), (g, R + 3)])
    assert (a[0].n, a[1].n) == O.g1_multiply(O.G1, 2)
    assert pb.ec_mul(g, pb.Scalar(5)) == O.g1_multiply(O.G1, 5)
    assert pb.ec_mul(None, 5) is None and pb.ec_lincomb([(g, 0)]) is None


def test_prove_rejects_non_canonical_arrays(pb, setup):
    """array inputs are canonical 32-byte little-endian field elements: a wire value or a public input >= r is refused
    (the list-of-ints surface reduces mod r like the reference's Scalar(...); raw arrays cannot be reduced silently)"""
    entry, arr = load_circuit("factorization")
    n = entry["n"]
    prover = pb.Prover.from_arrays(setup, n, _pk(arr))
    good = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    rows = lambda v: np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in v), dtype=np.uint8).reshape(-1, 32).copy()  # noqa: E731
    A = rows(arr["A"])
    A = np.concatenate([A, np.zeros((n - A.shape[0], 32), dtype=np.uint8)])
    bad = A.copy()
    bad[1] = np.frombuffer((int.from_bytes(bytes(A[1]), "little") + R).to_bytes(32, "little"), dtype=np.uint8)  # same residue, not reduced
    from plonkathon_b200._lib import PlonkB200Error
    with pytest.raises(PlonkB200Error, match="not reduced"):
        prover.prove_arrays(bad, arr["B"], arr["C"], ints(entry["public"]))
    pub = rows(ints(entry["public"]))
    pub_bad = pub.copy()
    pub_bad[0] = np.frombuffer((int.from_bytes(bytes(pub[0]), "little") + R).to_bytes(32, "little"), dtype=np.uint8)
    with pytest.raises(PlonkB200Error, match="not reduced"):
        prover.prove_arrays(A, arr["B"], arr["C"], pub_bad)
    assert prover.prove_arrays(A, arr["B"], arr["C"], pub) == good  # the prover object is fine afterwards


def test_prove_2p22_gates_runs(pb):
    """BASELINE.json's largest configuration size (2^22 gates, 4n = 2^24 domain: the three-pass NTT) on one GPU: the
    proof is deterministic, and its commitments are exact -- the fixed-base MSM at its widest window (c = 21), batched
    over 2 and 3 vectors as the prover commits them: a, b, c, z from the prover's Lagrange values and t_lo, t_mid,
    t_hi from its quotient coefficients, each [f(tau)]G with f evaluated on the host (oracle/c); the verifier accepts
    the proof, which with every other commitment exact pins W_z and W_zw too."""
    import torch
    if torch.cuda.get_device_properties(0).total_memory < 60 * 2 ** 30:
        pytest.skip("needs ~40 GB of HBM")
    from oracle import c_oracle as Co
    from plonkathon_b200 import _lib, synthetic as syn
    log_n = 22
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=9, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    bucket_c = ctypes.c_uint(0)
    _lib.check(_lib.lib().pb200_srs_bucket_count(setup._srs, ctypes.byref(bucket_c)))
    assert bucket_c.value == 1 << 20  # c = 21
    prover = pb.Prover.from_arrays(setup, n, pk)
    raw = prover.prove_arrays(A, B, C, public)
    assert prover.prove_arrays(A, B, C, public) == raw
    proof = O.proof_from_bytes(raw)

    def state(which):
        t = torch.empty((n, 32), dtype=torch.uint8, device="cuda")
        _lib.check(_lib.lib().pb200_prover_read_vector(prover._h, which, ctypes.c_void_p(t.data_ptr())))
        return t.cpu().numpy()

    for which, key in enumerate(("a_1", "b_1", "c_1", "z_1")):  # Lagrange values
        assert proof[key] == O.g1_multiply(O.G1, Co.eval_lagrange(state(which), TAU)), key
    for which, key in zip((5, 6, 7), ("t_lo_1", "t_mid_1", "t_hi_1")):  # coefficients
        assert proof[key] == O.g1_multiply(O.G1, Co.eval_coeffs(state(which), TAU)), key
    vk = setup.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), pub)
    k = 32 * 19  # z_shifted_eval
    raw_bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not vk.verify_proof(n, pb.Proof.from_bytes(raw_bad), pub)


# ------------------------------------------------------------------ exact full-size parity vs the C oracle
@pytest.mark.parametrize("logn", [20])
def test_ntt_2p20_exact_vs_c_oracle(pb, logn):
    """BASELINE.json configs[1]: Fr NTT forward + inverse at 2^20, every element compared with the C
    restatement of poly.py:113-149 (oracle/c/plonk_oracle.c, itself checked against the pinned Python oracle)"""
    from oracle import c_oracle as C
    n = 1 << logn
    x = _random_fr(n, 42)
    xb = x.view(np.uint8).reshape(n, 32)
    assert np.array_equal(_raw_ntt(pb, x, logn, 0).view(np.uint8).reshape(n, 32), C.fft(xb, False))
    assert np.array_equal(_raw_ntt(pb, x, logn, 1).view(np.uint8).reshape(n, 32), C.fft(xb, True))


def test_msm_2p20_distinct_points_exact_vs_c_oracle(pb):
    """BASELINE.json configs[2]: KZG G1 MSM over 2^20 DISTINCT points (structured SRS exported from the device)
    with uniform scalars, both MSM modes, bit-exact against the C restatement of curve.py:38-44"""
    from oracle import c_oracle as C
    from plonkathon_b200 import _lib
    n = 1 << 20
    setup = pb.Setup.generate(TAU, n)
    buf = ctypes.create_string_buffer(64 * n)
    _lib.check(_lib.lib().pb200_srs_export(setup.ctx.handle, setup._srs, buf, 0, n))
    pts = np.frombuffer(buf.raw, dtype=np.uint8).reshape(n, 64)
    sc = _random_fr(n, 77)
    exp = C.g1_lincomb(pts, sc.view(np.uint8).reshape(n, 32))
    out = ctypes.create_string_buffer(64)
    ident = ctypes.c_int(0)
    _lib.check(_lib.lib().pb200_g1_msm_host(setup.ctx.handle, pts.ctypes.data_as(ctypes.c_void_p),
                                            sc.ctypes.data_as(ctypes.c_void_p), n, out, ctypes.byref(ident)))
    assert (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little")) == exp
    import torch
    dev = torch.from_numpy(sc.view(np.int32)).cuda()
    _lib.check(_lib.lib().pb200_srs_commit_coeffs(setup.ctx.handle, setup._srs, ctypes.c_void_p(dev.data_ptr()), n, 0,
                                                  out, ctypes.byref(ident)))
    assert (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little")) == exp


def test_polynomial_results_stay_device_resident(pb, setup):
    """transform results keep their data in HBM and materialise list[Scalar] lazily; chains and commit agree
    with the oracle"""
    rng = random.Random(8)
    v = [rng.randrange(R) for _ in range(256)]
    p = pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE)
    c = p.ifft()
    assert c._values is None and len(c) == 256  # nothing crossed back yet
    back = c.fft()
    assert back == p and vals(c) == O.ifft(v)
    off = pb.Scalar(rng.randrange(1, R))
    ext = p.to_coset_extended_lagrange(off)
    assert len(ext) == 1024 and vals(ext.coset_extended_lagrange_to_coeffs(off))[:256] == O.ifft(v)
    got = setup.commit(c.fft())  # device-resident input
    assert (got[0].n, got[1].n) == O.Setup.from_file(PTAU_HEAD).commit(v)
    c.values = S(pb, [1, 2, 3, 4])  # assigning values drops the device copy
    assert len(c) == 4 and vals(c.fft()) == O.fft([1, 2, 3, 4])


# ------------------------------------------------------------------ more of the reference surface
class _CellProgram:
    """Program-shaped object (group_order, common_preprocessed_input, wires, get_public_assignments) built from
    a fixture: every cell gets its own variable name, the witness maps names to the fixture's wire values."""

    def __init__(self, pb, entry, arr):
        from collections import namedtuple
        self.group_order = entry["n"]
        self._W = namedtuple("GateWires", "L R O")
        self._PK = namedtuple("PK", "group_order QM QL QR QO QC S1 S2 S3")
        self._P = namedtuple("Poly", "values")
        self._pb, self._arr = pb, arr
        self.n_public = len(entry["public"])
        self.rows = len(arr["A"])

    def common_preprocessed_input(self):
        a = self._arr
        return self._PK(self.group_order, *[self._P([self._pb.Scalar(v) for v in a[k]])
                                            for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")])

    def wires(self):
        return [self._W("L%d" % i, "R%d" % i, "O%d" % i) for i in range(self.rows)]

    def get_public_assignments(self):
        return ["L%d" % i for i in range(self.n_public)]  # public rows carry the variable on the left wire

    def witness(self):
        a = self._arr
        w = {}
        for i in range(self.rows):
            w["L%d" % i], w["R%d" % i], w["O%d" % i] = a["A"][i], a["B"][i], a["C"][i]
        return w


@pytest.mark.parametrize("name", ["factorization", "poseidon"])
def test_round_by_round_surface_equals_one_call(pb, setup, name):
    """Prover(setup, program).prove(witness) -- round_1..5 driven from Python with the Transcript class, as the
    reference's prove() does -- gives the fixture proof, i.e. the same bytes as the single C call"""
    import hashlib
    entry, arr = load_circuit(name)
    prog = _CellProgram(pb, entry, arr)
    proof = pb.Prover(setup, prog).prove(prog.witness())
    assert hashlib.sha256(proof.to_bytes()).hexdigest() == entry["proof_sha256"]
    flat = proof.flatten()
    assert list(flat) == list(entry["proof"])  # prover.py:18-35 field order


def test_prover_rejects_broken_permutation(pb, setup):
    """a permutation that does not match the wiring: gates still hold, the grand product does not close
    (prover.py:132 assert Z_values.pop() == 1)"""
    entry, arr = load_circuit("factorization")
    pk = _pk(arr)
    pk = dict(pk)
    s1 = list(pk["S1"])
    s1[1], s1[2] = s1[2], s1[1]
    s1[3] = (s1[3] + 1) % R
    pk["S1"] = s1
    prover = pb.Prover.from_arrays(setup, entry["n"], pk)
    with pytest.raises(AssertionError, match="grand product"):
        prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))


def test_random_small_ntt_and_msm_property(pb):
    """hypothesis: random sizes / values incl. the field's edge values, NTT and ec_lincomb vs the oracle"""
    from hypothesis import given, settings, strategies as st, HealthCheck
    edge = st.sampled_from([0, 1, 2, R - 1, R - 2, (R - 1) // 2, 1 << 253, (1 << 32) - 1, 1 << 64])
    elem = st.one_of(edge, st.integers(min_value=0, max_value=R - 1))
    osetup = O.Setup.from_file(PTAU_HEAD)

    @settings(max_examples=25, deadline=None, suppress_health_check=list(HealthCheck))
    @given(st.integers(min_value=0, max_value=7).flatmap(lambda k: st.lists(elem, min_size=1 << k, max_size=1 << k)))
    def ntt(v):
        assert vals(pb.Polynomial(S(pb, v), pb.Basis.MONOMIAL).fft()) == O.fft(v)
        assert vals(pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE).ifft()) == O.ifft(v)

    @settings(max_examples=20, deadline=None, suppress_health_check=list(HealthCheck))
    @given(st.lists(st.tuples(st.integers(min_value=0, max_value=40), st.one_of(edge, st.integers(-5, R + 5))),
                    min_size=1, max_size=24))
    def msm(pairs):
        pts = osetup.powers_of_x
        got = pb.ec_lincomb([((pb.FQ(pts[i][0]), pb.FQ(pts[i][1])), s) for i, s in pairs])
        exp = O.ec_lincomb_naive([(pts[i], s % R) for i, s in pairs])
        assert (got is None and exp is None) or (got[0].n, got[1].n) == exp

    ntt()
    msm()


@pytest.mark.parametrize("seed", range(8))
def test_prove_random_circuits_vs_oracle(pb, seed):
    """differential test over randomly shaped circuits of the synthetic family: group orders 2^3..2^6, partly
    filled, 0..3 public inputs -- proof bytes equal the oracle's"""
    from plonkathon_b200 import synthetic as syn
    rng = random.Random(1000 + seed)
    log_n = rng.randrange(3, 7)
    n = 1 << log_n
    n_public = rng.randrange(0, 4)
    fill = rng.choice([1.0, 0.9, 0.6])
    c = syn.build_circuit(log_n, seed=seed, n_public=n_public, fill=fill)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU + seed, n)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, C, public)
    S1, S2, S3 = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    opk = O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3)
    osetup = O.Setup([(p[0].n, p[1].n) for p in setup.powers_of_x], None)
    a, b, cc = c.wires_values()
    assert raw == O.proof_bytes(O.Prover(osetup, opk).prove(a, b, cc, c.public_values())), (log_n, n_public, fill)


def _golden_vk(pb, entry):
    v = entry["vk"]
    x2 = (pb.FQ2([int(c) for c in v["X_2"][0]]), pb.FQ2([int(c) for c in v["X_2"][1]]))
    return pb.VerificationKey(entry["n"], *[pt(v[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")],
                              x2, pb.Scalar(int(v["w"])))


@pytest.mark.parametrize("name", ["prover_test", "factorization", "poseidon"])
def test_verifier_on_golden_proofs(pb, name):
    """verifier.py:40-92 completed (SURVEY 8(f) N3): the golden proofs -- accepted by the reference's own
    TESTING verifier when the fixtures were generated -- verify through GPU ec_lincomb + the library's pairing;
    tampered proofs and wrong public inputs do not"""
    entry, _ = load_circuit(name)
    vk = _golden_vk(pb, entry)
    n, public = entry["n"], [int(x) for x in entry["public"]]
    raw = O.proof_bytes({k: (pt(val) if isinstance(val, list) else int(val)) for k, val in entry["proof"].items()})
    proof = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(n, proof, public) and vk.verify_proof_unoptimized(n, proof, public)
    assert not vk.verify_proof(n, proof, [public[0] + 1] + public[1:])
    for word in (14, 17, 19):  # a_eval, s1_eval, z_shifted_eval
        k = 32 * word
        bad = pb.Proof.from_bytes(raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:])
        assert not vk.verify_proof(n, bad, public) and not vk.verify_proof_unoptimized(n, bad, public)
    swapped = pb.Proof.from_bytes(raw[:32 * 20] + raw[32 * 22:] + raw[32 * 20:32 * 22])  # W_z <-> W_zw
    assert not vk.verify_proof(n, swapped, public) and not vk.verify_proof_unoptimized(n, swapped, public)


def test_prove_then_verify_like_reference_test(pb, setup):
    """test.py:105-133 (prover_test_dummy_verifier) end to end on the product: Setup.from_file -> Prover.prove
    -> Setup.verification_key -> both verification routines"""
    from collections import namedtuple
    entry, arr = load_circuit("prover_test")
    PK = namedtuple("PK", "group_order QM QL QR QO QC S1 S2 S3")
    cols = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")
    pk = PK(8, *[pb.Polynomial(S(pb, arr[k]), pb.Basis.LAGRANGE) for k in cols])
    prover = pb.Prover.from_arrays(setup, 8, {k: arr[k] for k in cols})
    raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], [int(x) for x in entry["public"]])
    vk = setup.verification_key(pk)
    assert vk.X_2 == _golden_vk(pb, entry).X_2
    proof = pb.Proof.from_bytes(raw)
    assert vk.verify_proof_unoptimized(8, proof, [60]) and vk.verify_proof(8, proof, [60])
    assert not vk.verify_proof(8, proof, [61])


def test_commit_through_ptau_lagrange_section(pb):
    """SURVEY 8(f) N4: with the .ptau's Lagrange-basis points (section 12) Setup.commit is one MSM over the values.
    Same results as the reference pins for the inverse-transform path: commitment KAT (test.py:23-28) and the
    snarkjs verification keys of the n = 8 circuits; n = 16 (factorization); sizes without a block fall back."""
    import os
    from collections import namedtuple
    from tests.golden_io import GOLDEN
    setup = pb.Setup.from_file(PTAU_HEAD)
    assert setup._lagrange_handle(8) is None  # the committed head of the file stops before section 12
    setup.load_lagrange_section(open(os.path.join(GOLDEN, "ptau_lagrange_p0_p4.bin"), "rb").read())
    kat = load_json("circuits.json")["commit_kat"]
    c = setup.commit(pb.Polynomial(S(pb, ints(kat["lagrange"])), pb.Basis.LAGRANGE))
    assert setup._lagrange_handle(8) is not None and (c[0].n, c[1].n) == pt(kat["point"])
    PK = namedtuple("PK", "group_order QM QL QR QO QC S1 S2 S3")
    cols = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")
    for name in ("basic", "ab_plus_a", "one_public", "prover_test", "factorization"):
        entry, arr = load_circuit(name)
        n = entry["n"]
        vk = setup.verification_key(PK(n, *[pb.Polynomial(S(pb, arr[k]), pb.Basis.LAGRANGE) for k in cols]))
        for key in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
            got, exp = getattr(vk, key), pt(entry["vk"][key])
            assert (got is None and exp is None) or (got[0].n, got[1].n) == exp, (name, key)
        assert setup._lagrange_handle(n) is not None
        vk2 = setup.verification_key_arrays(n, {k: np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in arr[k]),
                                                                 dtype=np.uint8).reshape(-1, 32) for k in cols})
        assert vk2 == vk
    rng = random.Random(5)
    v = [rng.randrange(R) for _ in range(32)]  # no 32-point block in the fixture: inverse transform + monomial powers
    c = setup.commit(pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE))
    assert setup._lagrange_handle(32) is None and (c[0].n, c[1].n) == O.Setup.from_file(PTAU_HEAD).commit(v)


def test_commit_through_generated_lagrange_srs(pb):
    """the same for a structured test SRS: [L_i(tau)]G generated on the device (inverse NTT of the tau powers, then
    fixed-base multiplication); commitments equal the inverse-transform path's and the direct evaluation f(tau) G"""
    n_max = 1 << 12
    setup = pb.Setup.generate(TAU, n_max)
    rng = random.Random(6)
    for n in (8, 256, n_max):
        v = [rng.randrange(R) for _ in range(n)]
        v[1] = 0
        poly = pb.Polynomial(S(pb, v), pb.Basis.LAGRANGE)
        via_ntt = setup.commit(poly)
        assert setup.enable_lagrange(n)
        via_lagrange = setup.commit(poly)
        assert via_lagrange == via_ntt
        assert (via_lagrange[0].n, via_lagrange[1].n) == O.g1_multiply(O.G1, O.eval_lagrange_at(v, TAU))
    from plonkathon_b200 import synthetic as syn
    c = syn.build_circuit(10, seed=3, n_public=1)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup.disable_lagrange()
    vk_ntt = setup.verification_key_arrays(1 << 10, pk)
    assert setup.enable_lagrange(1 << 10)
    assert setup.verification_key_arrays(1 << 10, pk) == vk_ntt
    raw = pb.Prover.from_arrays(setup, 1 << 10, pk).prove_arrays(A, B, C, public)
    assert vk_ntt.verify_proof(1 << 10, pb.Proof.from_bytes(raw), [int(x) for x in public])


def test_two_prover_lanes_on_one_gpu(pb):
    """bench.py's throughput mode: two provers on their own contexts (stream + scratch), sharing one SRS, driven from
    two host threads at the same time -- same bytes as one prover alone, every time"""
    from concurrent.futures import ThreadPoolExecutor
    from plonkathon_b200 import _lib, synthetic as syn
    log_n = 14
    n = 1 << log_n
    setup = pb.Setup.generate(TAU, n)
    circuits = [syn.circuit_arrays(syn.build_circuit(log_n, seed=s, n_public=2)) for s in (11, 12)]
    alone = [pb.Prover.from_arrays(setup, n, c[0]).prove_arrays(c[1], c[2], c[3], c[4]) for c in circuits]
    assert alone[0] != alone[1]
    lanes = [pb.Prover.from_arrays(setup, n, c[0], ctx=_lib.Context(0) if i else None) for i, c in enumerate(circuits)]
    assert lanes[0].ctx is setup.ctx and lanes[1].ctx is not setup.ctx

    def worker(i):
        c = circuits[i]
        return [lanes[i].prove_arrays(c[1], c[2], c[3], c[4]) for _ in range(6)]

    with ThreadPoolExecutor(2) as pool:
        got = list(pool.map(worker, range(2)))
    assert got[0] == [alone[0]] * 6 and got[1] == [alone[1]] * 6


@pytest.mark.skipif(__import__("os").environ.get("PB200_TEST_2P22") != "1",
                    reason="opt-in (PB200_TEST_2P22=1): BASELINE.json's largest configuration, ~1 minute and 25 GB of HBM")
def test_prove_2p22_gates_against_golden(pb):
    """2^22 gates (4n = 2^24: the three-pass NTT): byte for byte against tests/golden/proof_2p22.json (oracle prover
    over the C restatement, ~2.5 CPU-hours) when that fixture has been generated, and accepted by the verifier"""
    import json
    import os
    from plonkathon_b200 import synthetic as syn
    from tests.golden_io import GOLDEN
    log_n = 22
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=7, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, C, public)
    path = os.path.join(GOLDEN, "proof_2p22.json")
    if os.path.exists(path):
        assert raw.hex() == json.load(open(path))["proof_hex"]
    vk = setup.verification_key_arrays(n, pk)
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), [int(x) for x in public])


# ------------------------------------------------------------------ ring operations and round state on the device
def test_polynomial_ring_ops_on_device(pb):
    """poly.py:23-109 on device-resident operands (pb200_fr_vec_op) against the reference's list arithmetic, which the
    same class runs for plain-list operands: + - * / with a Polynomial or a Scalar, both bases, shift; a zero divisor
    gives 0 (py_ecc's inv(0) == 0); mixed resident / list operands; in-place edits of .values are seen afterwards"""
    rng = random.Random(21)
    n = 1 << 10
    va = [rng.randrange(R) for _ in range(n)]
    vb = [rng.randrange(R) for _ in range(n)]
    vb[3] = vb[700] = 0
    s = pb.Scalar(rng.randrange(1, R))
    L, M = pb.Basis.LAGRANGE, pb.Basis.MONOMIAL

    def resident(v, basis):  # a Polynomial whose data lives in HBM only (the result of a transform)
        p = pb.Polynomial(S(pb, v), basis)
        q = p.ifft().fft() if basis == L else p.fft().ifft()  # round trip: same values, device-resident
        assert q._values is None and q.on_device and q.basis == basis
        return q

    for basis in (L, M):
        la, lb = pb.Polynomial(S(pb, va), basis), pb.Polynomial(S(pb, vb), basis)
        ops = [lambda x, y: x + y, lambda x, y: x - y, lambda x, y: x + s, lambda x, y: x - s, lambda x, y: x * s,
               lambda x, y: x / s, lambda x, y: x / pb.Scalar(0)]
        if basis == L:
            ops += [lambda x, y: x * y, lambda x, y: x / y, lambda x, y: x.shift(5), lambda x, y: x.shift(0),
                    lambda x, y: (x * y + x * s - y) / (y + s)]
        for k, op in enumerate(ops):
            want = op(la, lb)
            assert not want.on_device
            for da, db in ((resident(va, basis), resident(vb, basis)), (resident(va, basis), lb), (la, resident(vb, basis))):
                got = op(da, db)
                if da.on_device:
                    assert got.on_device and got._values is None, k
                assert got.basis == basis and got == want and vals(got) == vals(want), (basis, k)
    with pytest.raises(AssertionError):
        resident(va, M) * resident(vb, M)  # element-wise product is a LAGRANGE-basis operation (poly.py:67)
    # the list is the source of truth once it has been handed out
    p = resident(va, L)
    p.values[0] = pb.Scalar(123)
    assert not p.on_device and vals(p.ifft().fft())[0] == 123


def test_reference_style_round_3_through_the_facade(pb):
    """prover.py:154-226 written the way the reference prescribes -- Polynomial arithmetic on the round state
    self.A .. self.Z, fft_expand / expanded_evals_to_coeffs / rlc (prover.py:308-315) -- on 4n = 2^16 device-resident
    values, against the library's own round 3: the same T1, T2, T3 (hence the same commitments), the degree check
    of prover.py:205-208 and the T1/T2/T3 identity of prover.py:215-219."""
    from plonkathon_b200 import synthetic as syn
    from plonkathon_b200.transcript import Transcript
    log_n = 14
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=5, n_public=3)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk)
    tr = Transcript(b"plonk")
    prover.beta, prover.gamma = tr.round_1(prover.round_1_arrays(A, B, C, public))
    prover.alpha, prover.fft_cofactor = tr.round_2(prover.round_2())
    msg_3 = prover.round_3()
    L = pb.Basis.LAGRANGE
    one = pb.Scalar(1)
    col = lambda k: pb.Polynomial([pb.Scalar(int.from_bytes(bytes(r), "little")) for r in pk[k]], L)  # noqa: E731
    roots = [pb.Scalar(x) for x in O.roots_of_unity(n)]
    # round state: device-resident Lagrange polynomials
    sA, sB, sC, sZ, sPI = prover.A, prover.B, prover.C, prover.Z, prover.PI
    assert all(p.on_device and p.basis == L and len(p) == n for p in (sA, sB, sC, sZ, sPI))
    assert sA == pb.Polynomial([pb.Scalar(int.from_bytes(bytes(r), "little")) for r in A], L)
    # the reference's round-1 sanity check (prover.py:108-116), on the device
    zero = pb.Polynomial([pb.Scalar(0)] * n, L)
    assert sA * col("QL") + sB * col("QR") + sA * sB * col("QM") + sC * col("QO") + sPI + col("QC") == zero
    ex = prover.fft_expand
    A_big, B_big, C_big, Z_big, PI_big = ex(sA), ex(sB), ex(sC), ex(sZ), ex(sPI)
    ZW_big = Z_big.shift(4)
    QL, QR, QM, QO, QC = (ex(col(k)) for k in ("QL", "QR", "QM", "QO", "QC"))
    S1, S2, S3 = (ex(col(k)) for k in ("S1", "S2", "S3"))
    cof = prover.fft_cofactor
    mu = pb.Scalar(O.root_of_unity(4 * n))
    quarter_roots = [cof * mu ** i for i in range(4 * n)]
    X_big = pb.Polynomial(quarter_roots, L)
    ZH_big = pb.Polynomial([x ** n - one for x in quarter_roots], L)
    L0_big = ex(pb.Polynomial([one] + [pb.Scalar(0)] * (n - 1), L))
    rlc, al = prover.rlc, prover.alpha
    gate = A_big * QL + B_big * QR + A_big * B_big * QM + C_big * QO + PI_big + QC
    perm = (rlc(A_big, X_big) * rlc(B_big, X_big * pb.Scalar(2)) * rlc(C_big, X_big * pb.Scalar(3))) * Z_big \
        - (rlc(A_big, S1) * rlc(B_big, S2) * rlc(C_big, S3)) * ZW_big
    QUOT_big = (gate + perm * al + (Z_big - one) * L0_big * (al * al)) / ZH_big
    assert QUOT_big.on_device and len(QUOT_big) == 4 * n
    coeffs = prover.expanded_evals_to_coeffs(QUOT_big)
    cv = vals(coeffs)
    assert cv[-n:] == [0] * n  # prover.py:205-208
    T1, T2, T3 = prover.T1, prover.T2, prover.T3  # the library's round 3, as the reference's Lagrange polynomials
    assert [vals(t.ifft()) for t in (T1, T2, T3)] == [cv[:n], cv[n:2 * n], cv[2 * n:3 * n]]
    assert (T1.barycentric_eval(cof) + T2.barycentric_eval(cof) * cof ** n
            + T3.barycentric_eval(cof) * cof ** (2 * n)) == QUOT_big.values[0]  # prover.py:215-219
    assert (setup.commit(T1), setup.commit(T2), setup.commit(T3)) == (msg_3.t_lo_1, msg_3.t_mid_1, msg_3.t_hi_1)
