"""Zero-knowledge proving: A, B, C, Z and the quotient pieces blinded as in the PLONK paper (tests/extended_oracle.py has the
construction), with the proof format, the transcript and the verifier unchanged.

CPU: the zero-knowledge oracle's proofs verify (trapdoor check and the product's host verifier) and tampered ones do not;
zero blinders give the plain oracle's bytes; different blinders change every commitment and evaluation; the blinded
quotient pieces recombine to T; custom gates work with blinding.  GPU: the prover's 768 bytes equal the oracle's with
fixed blinders; zero blinders reproduce the existing golden proofs; the 2^16 zero-knowledge golden proof is reproduced;
proofs with fresh OS randomness differ and verify; the limits are refused with messages that name them."""
import json
import os
import random

import numpy as np
import pytest

from oracle import fast as F
from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from tests import extended_oracle as XO
from tests.oracle_keys import host_lincomb  # noqa: F401  (a fixture)
from tests.golden_io import GOLDEN, PTAU_HEAD, ints, load_circuit, pt

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
ALL_TERMS = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]
PK_KEYS = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")
VK_KEYS = (("Qm", "QM"), ("Ql", "QL"), ("Qr", "QR"), ("Qo", "QO"), ("Qc", "QC"), ("S1", "S1"), ("S2", "S2"), ("S3", "S3"))
COMMITMENTS = ("a_1", "b_1", "c_1", "z_1", "t_lo_1", "t_mid_1", "t_hi_1", "W_z_1", "W_zw_1")
EVALUATIONS = ("a_eval", "b_eval", "c_eval", "s1_eval", "s2_eval", "z_shifted_eval")


def _blinders(seed):
    rng = random.Random(seed)
    return [rng.randrange(1, R) for _ in range(11)]


def _custom_circuit(log_n, n_public, seed):
    """the first circuit from ``seed`` on whose rows every custom term is used"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=ALL_TERMS)
        if all(any(col) for _, col in c.custom):
            return c
        seed += 1000


def _oracle(c, blinders, fast=True):
    """(pk, fast setup of n + 6 powers, oracle zero-knowledge proof, prover object) of a synthetic circuit"""
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    fsetup = F.Setup(TAU, n + 6)
    setup = fsetup if fast else O.Setup([fsetup.point(i) for i in range(n + 6)], None)
    prover = XO.Prover(setup, pk, blinders)
    if fast:
        with F.c_kernels():
            proof = prover.prove(A, B, C, c.public_values())
    else:
        proof = prover.prove(A, B, C, c.public_values())
    return pk, fsetup, proof, prover


def _oracle_vk(pk, fsetup):
    with F.c_kernels():
        vk = {k: fsetup.commit(getattr(pk, a)) for k, a in VK_KEYS}
        custom = [(e, fsetup.commit(col)) for e, col in getattr(pk, "custom", ())]
    return vk, custom


# ---- CPU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n", [3, 4, 6, 8])
def test_oracle_zk_proof_verifies(log_n, host_lincomb):
    pb = host_lincomb
    c = syn.build_circuit(log_n, seed=40 + log_n, n_public=2)
    n = c.group_order
    pk, fsetup, proof, _ = _oracle(c, _blinders(log_n), fast=log_n > 4)  # n = 8, 16: the pure-Python oracle
    vk, _ = _oracle_vk(pk, fsetup)
    public = c.public_values()
    assert O.verify_proof_trapdoor(n, vk, proof, public, TAU)
    bad_eval = dict(proof, b_eval=(proof["b_eval"] + 1) % R)
    swapped = dict(proof, W_z_1=proof["W_zw_1"], W_zw_1=proof["W_z_1"])
    assert not O.verify_proof_trapdoor(n, vk, bad_eval, public, TAU)
    assert not O.verify_proof_trapdoor(n, vk, swapped, public, TAU)
    # the product's verifier, unchanged, with its pairing against X2 = [tau]_2
    fq = lambda p: None if p is None else (pb.FQ(p[0]), pb.FQ(p[1]))  # noqa: E731  (None: an all-zero selector)
    key = pb.VerificationKey(n, *[fq(vk[k]) for k, _ in VK_KEYS], pb.g2_mul(pb.G2, TAU), pb.Scalar.root_of_unity(n))
    for p, ok in ((proof, True), (bad_eval, False), (swapped, False)):
        pf = pb.Proof.from_bytes(O.proof_bytes(p))
        assert key.verify_proof(n, pf, public) is ok
        assert key.verify_proof_unoptimized(n, pf, public) is ok


def test_oracle_zero_blinders_give_the_plain_proof():
    """the reference's test/proof.pickle circuit on the shipped .ptau, and a synthetic circuit"""
    entry, arr = load_circuit("prover_test")
    osetup = O.Setup.from_file(PTAU_HEAD)
    opk = XO.Preprocessed(entry["n"], *[arr[k] for k in PK_KEYS])
    public = ints(entry["public"])
    zk = XO.prove(osetup, opk, arr["A"], arr["B"], arr["C"], public, [0] * 11)
    plain = O.Prover(osetup, opk).prove(arr["A"], arr["B"], arr["C"], public)
    assert O.proof_bytes(zk) == O.proof_bytes(plain)
    assert all(((pt(v) if isinstance(v, list) else int(v)) == zk[k]) for k, v in entry["proof"].items())
    c = syn.build_circuit(6, seed=9, n_public=3)
    n = c.group_order
    pk, fsetup, zk, _ = _oracle(c, [0] * 11)
    A, B, C = c.wires_values()
    assert zk == F.prove(fsetup, pk, A, B, C, c.public_values())


def test_oracle_different_blinders_change_every_value():
    c = syn.build_circuit(5, seed=3, n_public=2)
    pk, fsetup, p1, _ = _oracle(c, _blinders(1))
    _, _, p2, _ = _oracle(c, _blinders(2))
    for k in COMMITMENTS + EVALUATIONS:
        assert p1[k] != p2[k], k
    vk, _ = _oracle_vk(pk, fsetup)
    assert O.verify_proof_trapdoor(c.group_order, vk, p1, c.public_values(), TAU)
    assert O.verify_proof_trapdoor(c.group_order, vk, p2, c.public_values(), TAU)


def test_oracle_blinded_pieces_recombine_to_the_quotient():
    c = syn.build_circuit(5, seed=11, n_public=2)
    n = c.group_order
    _, _, _, prover = _oracle(c, _blinders(5))
    assert len(prover.T1b) == n + 1 and len(prover.T2b) == n + 1 and len(prover.T3b) == n + 6
    assert any(prover.T[3 * n:])  # the blinded quotient reaches past 3n
    x = random.Random(7).randrange(R)
    xn = pow(x, n, R)
    got = (XO.poly_eval(prover.T1b, x) + xn * XO.poly_eval(prover.T2b, x) + xn * xn * XO.poly_eval(prover.T3b, x)) % R
    assert got == XO.poly_eval(prover.T, x)


def test_oracle_custom_gates_with_zero_knowledge():
    c = _custom_circuit(6, 2, 60)
    n = c.group_order
    pk, fsetup, proof, _ = _oracle(c, _blinders(6))
    vk, custom = _oracle_vk(pk, fsetup)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=custom), proof, public, TAU)
    assert not XO.verify_proof_trapdoor(n, dict(vk, custom=custom), dict(proof, a_eval=(proof["a_eval"] + 1) % R), public, TAU)


def test_set_zk_argument_checks():
    import plonkathon_b200 as pb
    from plonkathon_b200 import parallel
    p = pb.Prover.__new__(pb.Prover)
    with pytest.raises(ValueError, match="11 blinders"):
        p.set_zk(True, [1] * 10)
    with pytest.raises(ValueError, match=r"\[0, r\)"):
        p.set_zk(True, [1] * 10 + [R])
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.__new__(parallel.ShardedProver).set_zk(True)


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _gpu_prover(pb, c, setup=None, blinders=None, zk=True):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n + 6)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c))
    if zk:
        prover.set_zk(True, blinders)
    return setup, pk, prover, (A, B, C, public)


@pytest.mark.gpu
@pytest.mark.parametrize("custom", [False, True], ids=["plain", "custom4"])
@pytest.mark.parametrize("log_n,n_public", [(4, 2), (8, 2), (12, 2), (8, 11), (12, 9)])
def test_gpu_zk_proof_equals_oracle(log_n, n_public, custom):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated (the two paths of k_quotient)"""
    import plonkathon_b200 as pb
    seed = 300 + log_n + n_public
    c = _custom_circuit(log_n, n_public, seed) if custom else syn.build_circuit(log_n, seed=seed, n_public=n_public)
    bl = _blinders(seed)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c, blinders=bl)
    raw = prover.prove_arrays(A, B, C, public)
    _, _, proof, _ = _oracle(c, bl)
    assert raw == O.proof_bytes(proof)
    assert prover.prove_arrays(A, B, C, public) == raw  # fixed blinders: the same proof again


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["prover_test", "factorization", "poseidon"])
def test_gpu_zero_blinders_reproduce_golden_proofs(name):
    import hashlib
    import plonkathon_b200 as pb
    entry, arr = load_circuit(name)
    setup = pb.Setup.from_file(PTAU_HEAD)
    prover = pb.Prover.from_arrays(setup, entry["n"], {k: arr[k] for k in PK_KEYS})
    prover.set_zk(True, [0] * 11)
    raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"]


@pytest.mark.gpu
def test_gpu_zk_2p20_zero_blinders_golden_and_fresh_blinders_verify():
    """zero blinders through the zero-knowledge path (n + 8 buffers, separate pieces, k_quotient<true>) at full size
    give the golden 2^20 proof; with fresh blinders the proof verifies by the trapdoor check and the product's verifier"""
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    c = syn.build_circuit(20, seed=rec["seed"], n_public=2)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c, blinders=[0] * 11)
    raw = prover.prove_arrays(A, B, C, public)
    assert raw.hex() == rec["proof_hex"], "zero-blinder proof differs from the golden 2^20 proof"
    prover.set_zk(True)
    raw = prover.prove_arrays(A, B, C, public)
    assert raw.hex() != rec["proof_hex"]
    vk = setup.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    pf = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)
    okey = {k: (getattr(vk, k)[0].n, getattr(vk, k)[1].n) for k, _ in VK_KEYS}
    proof = O.proof_from_bytes(raw)
    assert O.verify_proof_trapdoor(n, okey, proof, pub, TAU)
    assert not O.verify_proof_trapdoor(n, okey, dict(proof, a_eval=(proof["a_eval"] + 1) % R), pub, TAU)


@pytest.mark.gpu
def test_gpu_golden_zk_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_zk_2p16.json")))
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"])
    n = c.group_order
    setup = pb.Setup.generate(TAU, rec["srs_powers"])
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c, setup, [int(b) for b in rec["blinders"]])
    raw = prover.prove_arrays(A, B, C, public)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden zero-knowledge proof"
    vk = setup.verification_key_arrays(n, pk)
    assert {k: (getattr(vk, k)[0].n, getattr(vk, k)[1].n) for k, _ in VK_KEYS} == {k: pt(v) for k, v in rec["vk"].items()}
    pf = pb.Proof.from_bytes(raw)
    pub = [int(x) for x in rec["public"]]
    assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)


def _tamper_eval(raw, k):
    return raw[:32 * k] + ((int.from_bytes(raw[32 * k:32 * k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[32 * k + 32:]


@pytest.mark.gpu
def test_gpu_fresh_blinders_differ_and_verify():
    import plonkathon_b200 as pb
    c = syn.build_circuit(10, seed=12, n_public=2)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c)
    p1 = prover.prove_arrays(A, B, C, public)
    p2 = prover.prove_arrays(A, B, C, public)
    assert p1 != p2
    f1, f2 = O.proof_from_bytes(p1), O.proof_from_bytes(p2)
    assert all(f1[k] != f2[k] for k in COMMITMENTS + EVALUATIONS)
    vk = setup.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    for raw in (p1, p2):
        pf = pb.Proof.from_bytes(raw)
        assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)
        bad = pb.Proof.from_bytes(_tamper_eval(raw, 14))  # a_eval
        assert not vk.verify_proof(n, bad, pub) and not vk.verify_proof_unoptimized(n, bad, pub)
    # the round-by-round surface draws its blinders in round 1 too
    from plonkathon_b200.transcript import Transcript
    tr = Transcript(b"plonk")
    m1 = prover.round_1_arrays(A, B, C, public)
    prover.beta, prover.gamma = tr.round_1(m1)
    m2 = prover.round_2()
    prover.alpha, prover.fft_cofactor = tr.round_2(m2)
    m3 = prover.round_3()
    prover.zeta = tr.round_3(m3)
    m4 = prover.round_4()
    prover.v = tr.round_4(m4)
    m5 = prover.round_5()
    pf = pb.Proof(m1, m2, m3, m4, m5)
    assert pf.to_bytes() not in (p1, p2)
    assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)


@pytest.mark.gpu
def test_gpu_mini_poseidon_on_the_shipped_ptau():
    import plonkathon_b200 as pb
    entry, arr = load_circuit("poseidon")
    n = entry["n"]
    setup = pb.Setup.from_file(PTAU_HEAD)
    pk = {k: arr[k] for k in PK_KEYS}
    prover = pb.Prover.from_arrays(setup, n, pk)
    prover.set_zk(True)
    public = ints(entry["public"])
    raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], public)
    assert raw != prover.prove_arrays(arr["A"], arr["B"], arr["C"], public)
    pkb = {k: np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in arr[k]), np.uint8).reshape(-1, 32)
           for k in PK_KEYS}
    vk = setup.verification_key_arrays(n, pkb)
    pf = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    assert not vk.verify_proof(n, pf, [public[0] + 1] + public[1:])


@pytest.mark.gpu
def test_gpu_refusals_and_unchanged_round_state():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, parallel
    c = syn.build_circuit(6, seed=8, n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    short = pb.Setup.generate(TAU, n)
    with pytest.raises(_lib.PlonkB200Error, match=r"n \+ 6"):
        pb.Prover.from_arrays(short, n, pk).set_zk(True)
    tiny = {k: np.zeros((4, 32), np.uint8) for k in PK_KEYS}
    with pytest.raises(_lib.PlonkB200Error, match="n >= 8"):
        pb.Prover.from_arrays(pb.Setup.generate(TAU, 64), 4, tiny).set_zk(True)
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.__new__(parallel.ShardedProver).set_zk(True)
    setup = pb.Setup.generate(TAU, n + 6)
    raw_checked = pb.Prover.from_arrays(setup, n, pk)
    with pytest.raises(_lib.PlonkB200Error, match="not reduced"):  # the library checks the raw blinders itself
        _lib.check(_lib.lib().pb200_prover_set_zk(raw_checked._h, 1, b"\xff" * 32 * 11))
    plain = pb.Prover.from_arrays(setup, n, pk)
    plain.prove_arrays(A, B, C, public)
    zk = pb.Prover.from_arrays(setup, n, pk)
    zk.set_zk(True)
    zk.prove_arrays(A, B, C, public)
    for name in ("A", "B", "C", "PI"):  # the unblinded Lagrange values, as in plain mode
        assert [x.n for x in getattr(zk, name).values] == [x.n for x in getattr(plain, name).values], name
    # Z depends on beta and gamma, which the blinded commitments change: it is the unblinded grand product for the
    # zero-knowledge proof's own challenges (round-by-round path), and the plain prover's Z with zero blinders
    from plonkathon_b200.transcript import Transcript
    tr = Transcript(b"plonk")
    zk.beta, zk.gamma = tr.round_1(zk.round_1_arrays(A, B, C, public))
    zk.round_2()
    S = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    oz = O.Prover(None, O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, *S), check=False)
    oz.A, oz.B, oz.C = c.wires_values()
    oz.beta, oz.gamma = zk.beta.n, zk.gamma.n
    oz.setup = type("NoCommit", (), {"commit": lambda self, v: None})()
    oz.round_2()
    assert [x.n for x in zk.Z.values] == oz.Z
    zk.set_zk(True, [0] * 11)
    zk.prove_arrays(A, B, C, public)
    assert [x.n for x in zk.Z.values] == [x.n for x in plain.Z.values]
    with pytest.raises(RuntimeError, match="T1"):
        zk.T1
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge"):
        zk._state(5, None)
    zk.set_zk(False)  # back to plain proofs
    assert zk.prove_arrays(A, B, C, public) == plain.prove_arrays(A, B, C, public)
    assert [x.n for x in zk.T1.values] == [x.n for x in plain.T1.values]
