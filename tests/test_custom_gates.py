"""Custom gates: selector columns Q_k for degree-2 and degree-3 wire terms a^i b^j c^l (plonkathon_b200/custom_gates.py).

CPU: the oracle with custom terms (tests/extended_oracle.py) proves circuits that its trapdoor verifier and the
product's host verifier accept, and rejects what it must; malformed terms are refused.  GPU: the prover's 768 bytes
equal the oracle's for single terms and all four together, at several sizes and on both public-input paths; the 2^16
golden proof is reproduced; a 2^20-gate custom circuit verifies; the sharded prover agrees with the single-GPU one."""
import ctypes
import dataclasses
import json
import os

import numpy as np
import pytest

from oracle import fast as F
from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from tests import extended_oracle as XO
from tests.oracle_keys import host_lincomb  # noqa: F401  (a fixture)
from tests.golden_io import GOLDEN, pt

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
ALL_TERMS = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]
TERM_SETS = [[e] for e in ALL_TERMS] + [ALL_TERMS]
TERM_IDS = ["x2", "z3", "x2y", "xyz", "all4"]


def _circuit(log_n, n_public, terms, seed):
    """the synthetic circuit of the first seed from ``seed`` on whose rows use every term (small circuits may miss one)"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=terms)
        if all(any(col) for _, col in c.custom):
            return c
        seed += 1000


def _oracle_proof(c, fast=True):
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n)
    if not fast:
        setup = O.Setup([setup.point(i) for i in range(n)], None)
    return pk, setup, XO.prove(setup, pk, A, B, C, c.public_values(), fast=fast)


def _oracle_vk(c, pk, setup):
    with F.c_kernels():
        vk = {k: setup.commit(col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                  ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
        custom = [(e, setup.commit(col)) for e, col in c.custom]
    return vk, custom


# ---- CPU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_custom_proof_verifies(terms, log_n):
    c = _circuit(log_n, 2, terms, 100 + log_n)
    pk, setup, proof = _oracle_proof(c, fast=log_n > 4)  # 2^4: the pure-Python transforms
    vk, custom = _oracle_vk(c, pk, setup)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(c.group_order, dict(vk, custom=custom), proof, public, TAU)
    assert not XO.verify_proof_trapdoor(c.group_order, dict(vk, custom=custom), proof, [public[0] + 1] + public[1:], TAU)
    bad = dict(proof, c_eval=(proof["c_eval"] + 1) % R)
    assert not XO.verify_proof_trapdoor(c.group_order, dict(vk, custom=custom), bad, public, TAU)


@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
def test_oracle_rejects_violated_custom_row(terms):
    c = _circuit(5, 2, terms, 3)
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    row = next(i for i in range(c.group_order) if any(col[i] for _, col in c.custom))
    C[row] = (C[row] + 1) % R  # every term here has c in its row's constraint (as output or as a factor)
    with pytest.raises(AssertionError, match="gate %d unsatisfied" % row):
        XO.prove(F.Setup(TAU, c.group_order), pk, A, B, C, c.public_values(), fast=True)


def test_oracle_zero_custom_columns_give_the_plain_proof():
    c = syn.build_circuit(6, seed=9, n_public=3)
    n = c.group_order
    S = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n)
    plain = F.prove(setup, O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, *S), A, B, C, c.public_values())
    zero = dataclasses.replace(c, custom=[(e, [0] * n) for e in ALL_TERMS])
    assert XO.prove(setup, XO.preprocessed(zero, S), A, B, C, c.public_values(), fast=True) == plain


def test_custom_keyword_off_keeps_the_plain_circuit():
    """the golden proofs of the synthetic family depend on the circuit: custom=() draws the same random numbers"""
    a = syn.build_circuit(9, seed=20260924, n_public=2)
    b = syn.build_circuit(9, seed=20260924, n_public=2, custom=())
    for f in dataclasses.fields(a):
        x, y = getattr(a, f.name), getattr(b, f.name)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f.name
    assert a.custom == []


def test_host_verifier_accepts_custom_proofs_and_rejects_wrong_keys(host_lincomb):
    pb = host_lincomb
    c = _circuit(4, 2, ALL_TERMS, 21)
    n = c.group_order
    pk, setup, proof = _oracle_proof(c)
    vk, custom = _oracle_vk(c, pk, setup)
    fq = lambda p: (pb.FQ(p[0]), pb.FQ(p[1]))  # noqa: E731
    base = [fq(vk[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")]
    x2, w = pb.g2_mul(pb.G2, TAU), pb.Scalar.root_of_unity(n)
    terms = tuple((e, fq(p)) for e, p in custom)
    good = pb.VerificationKey(n, *base, x2, w, terms)
    pf = pb.Proof.from_bytes(O.proof_bytes(proof))
    public = c.public_values()
    assert good.verify_proof(n, pf, public) and good.verify_proof_unoptimized(n, pf, public)
    assert good != pb.VerificationKey(n, *base, x2, w)
    wrong = {
        "drop a term": terms[:3],
        "swap two commitments": ((terms[0][0], terms[1][1]), (terms[1][0], terms[0][1])) + terms[2:],
        "change a triple": (((3, 0, 0), terms[0][1]),) + terms[1:],
    }
    for why, t in wrong.items():
        vk_bad = pb.VerificationKey(n, *base, x2, w, t)
        assert not vk_bad.verify_proof(n, pf, public), why
        assert not vk_bad.verify_proof_unoptimized(n, pf, public), why


@pytest.mark.parametrize("terms,match", [
    ([(1, 0, 0)], "degree"), ([(0, 0, 1)], "degree"), ([(2, 2, 0)], "degree"), ([(4, 0, 0)], "degree"),
    ([(0, 0, 0)], "degree"), ([(1, 1, 0)], "QM"), ([(2, 0, 0), (2, 0, 0)], "twice"),
    ([(2, 0, 0), (0, 2, 0), (0, 0, 2), (3, 0, 0), (0, 3, 0)], "at most 4"), ([(1, -1, 2)], "non-negative"),
])
def test_malformed_terms_are_rejected(terms, match):
    import plonkathon_b200 as pb
    n = 16
    pk = {k: np.zeros((n, 32), np.uint8) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")}
    custom = [(e, np.zeros((n, 32), np.uint8)) for e in terms]
    with pytest.raises(ValueError, match=match):
        pb.Prover.from_arrays(None, n, pk, custom=custom)
    with pytest.raises(ValueError, match=match):
        pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, custom=custom)
    with pytest.raises(ValueError, match=match):
        syn.build_circuit(4, custom=terms)


def test_wrong_column_length_is_rejected():
    import plonkathon_b200 as pb
    n = 16
    pk = {k: np.zeros((n, 32), np.uint8) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")}
    with pytest.raises(ValueError, match="rows"):
        pb.Prover.from_arrays(None, n, pk, custom=[((2, 0, 0), np.zeros((n // 2, 32), np.uint8))])


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _gpu_proof(pb, c, setup=None):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c))
    return setup, pk, prover, prover.prove_arrays(A, B, C, public)


@pytest.mark.gpu
@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n,n_public", [(4, 2), (8, 2), (12, 2), (8, 11), (12, 9)])
def test_gpu_custom_proof_equals_oracle(terms, log_n, n_public):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated (the two paths of k_quotient)"""
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, terms, 200 + log_n + n_public)
    _, _, _, raw = _gpu_proof(pb, c)
    _, _, proof = _oracle_proof(c)
    assert raw == O.proof_bytes(proof)


@pytest.mark.gpu
def test_gpu_zero_terms_through_custom_entry_point():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    c = syn.build_circuit(8, seed=31, n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    plain = pb.Prover.from_arrays(setup, n, pk)
    h = ctypes.c_void_p()
    keep = [pk[k].tobytes() for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")]
    arr = (ctypes.c_char_p * 8)(*keep)
    _lib.check(_lib.lib().pb200_prover_create_custom(setup.ctx.handle, setup._srs, 8, ctypes.cast(arr, ctypes.c_void_p),
                                                     0, None, None, ctypes.byref(h)))
    via_custom = pb.Prover.__new__(pb.Prover)
    via_custom.group_order, via_custom.ctx, via_custom._h = n, setup.ctx, h
    assert via_custom.prove_arrays(A, B, C, public) == plain.prove_arrays(A, B, C, public)
    # and a malformed triple is refused by the library itself
    bad = ctypes.c_void_p()
    col = (ctypes.c_char_p * 1)(keep[0])
    rc = _lib.lib().pb200_prover_create_custom(setup.ctx.handle, setup._srs, 8, ctypes.cast(arr, ctypes.c_void_p), 1,
                                               bytes([1, 1, 0]), ctypes.cast(col, ctypes.c_void_p), ctypes.byref(bad))
    assert rc != 0 and "QM" in _lib.lib().pb200_last_error().decode()


@pytest.mark.gpu
def test_gpu_golden_custom_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_custom_2p16.json")))
    terms = [tuple(e) for e in rec["terms"]]
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"], custom=terms)
    n = c.group_order
    setup, pk, _, raw = _gpu_proof(pb, c)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden custom-gate proof"
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c))
    assert [(e, (p[0].n, p[1].n)) for e, p in vk.custom] == [(tuple(e), pt(p)) for e, p in rec["vk_custom"]]
    public = [int(x) for x in rec["public"]]
    pf = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_custom_2p20_verifies():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, custom=ALL_TERMS)
    n = c.group_order
    setup, pk, prover, raw = _gpu_proof(pb, c)
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c))
    public = c.public_values()
    pf = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public)
    # the trapdoor check of the oracle, with the key's commitments
    okey = {k: (getattr(vk, a)[0].n, getattr(vk, a)[1].n) for k, a in (
        ("Qm", "Qm"), ("Ql", "Ql"), ("Qr", "Qr"), ("Qo", "Qo"), ("Qc", "Qc"), ("S1", "S1"), ("S2", "S2"), ("S3", "S3"))}
    ocustom = [(e, (p[0].n, p[1].n)) for e, p in vk.custom]
    proof = O.proof_from_bytes(raw)
    assert XO.verify_proof_trapdoor(n, dict(okey, custom=ocustom), proof, public, TAU)
    # one custom commitment re-derived on the CPU: [Q_k(tau)] G
    e0, col0 = c.custom[0]
    assert ocustom[0][1] == O.g1_multiply(O.G1, O.eval_lagrange_at(col0, TAU))
    k = 32 * 16  # c_eval
    bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not vk.verify_proof(n, pb.Proof.from_bytes(bad), public)
    assert not XO.verify_proof_trapdoor(n, dict(okey, custom=ocustom), O.proof_from_bytes(bad), public, TAU)


@pytest.mark.gpu
def test_gpu_violated_custom_row_raises():
    import plonkathon_b200 as pb
    c = syn.build_circuit(10, seed=5, n_public=2, custom=ALL_TERMS)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    prover = pb.Prover.from_arrays(pb.Setup.generate(TAU, n), n, pk, custom=syn.custom_arrays(c))
    for e, col in c.custom:
        row = next(i for i in range(n) if col[i])
        bad = A.copy()
        bad[row, 0] ^= 1
        with pytest.raises(AssertionError, match="gate constraints"):
            prover.prove_arrays(bad, B, C, public)
    assert prover.prove_arrays(A, B, C, public)  # the prover is still usable


def _sharded_worker(rank, world, port, q):
    from tests.test_gpu_multi import _init
    torch, dist = _init(rank, world, port)
    import plonkathon_b200 as pb
    from plonkathon_b200 import parallel
    c = syn.build_circuit(12, seed=13, n_public=2, custom=ALL_TERMS)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    custom = syn.custom_arrays(c)
    single = pb.Prover.from_arrays(setup, n, pk, custom=custom).prove_arrays(A, B, C, public)
    sharded = parallel.ShardedProver.from_arrays(setup, n, pk, custom=custom).prove_arrays(A, B, C, public)
    q.put((rank, single == sharded))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_gpu_sharded_custom_proof_equals_single_gpu():
    from tests.test_gpu_multi import _spawn
    res = _spawn(_sharded_worker, 2)
    assert all(ok for _, ok in res), res
