"""Custom gates over the next row: terms Q_k a^i b^j c^l a(wX)^i' b(wX)^j' c(wX)^l' (plonkathon_b200/custom_gates.py).

CPU: exponent validation; the refusals of next-row terms with lookups and on the sharded prover; the oracle with
next-row terms (tests/extended_oracle.py) proves circuits at n = 16, 64 and 256 that its trapdoor verifier and both host
verifier routines accept, and both routines reject what they must; the gate check reads row 0 from row n - 1; the
zero-knowledge oracle with random blinders verifies.  GPU: the prover's 864 bytes equal the oracle's for each kind of
term and all four together, plain and in zero-knowledge mode, at several sizes and on both public-input paths; the
round-by-round ABI gives the same bytes; the 2^16 golden proof is reproduced; a 2^20 proof verifies; the library
refuses what it must."""
import ctypes
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
from tests.golden_io import GOLDEN, pt

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
# one term of each kind: degree 1 on the next row, a same-row wire times a next-row wire, degree 3 over the next row
# only, and a term over all of a, b, c and one next-row wire
ALL_TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
TERM_SETS = [[e] for e in ALL_TERMS] + [ALL_TERMS, list(syn.RUNNING_SUM_TERMS)]
TERM_IDS = ["a'", "aa'", "b'2c'", "bcc'", "all4", "running_sum"]
PK_KEYS = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")


def _circuit(log_n, n_public, terms, seed):
    """the synthetic circuit of the first seed from ``seed`` on whose rows use every term (small circuits may miss one)"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=terms)
        if all(any(col) for _, col in c.custom):
            return c
        seed += 1000


def _blinders(seed):
    rng = random.Random(seed)
    return [rng.randrange(R) for _ in range(14)]


def _oracle_proof(c, blinders=None, fast=True):
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n + 9)
    if not fast:
        setup = O.Setup([setup.point(i) for i in range(n + 9)], None)
    return pk, setup, XO.prove(setup, pk, A, B, C, c.public_values(), blinders=blinders, fast=fast)


def _oracle_vk(c, pk):
    setup = F.Setup(TAU, c.group_order)
    with F.c_kernels():
        vk = {k: setup.commit(col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                  ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
        custom = [(e, setup.commit(col)) for e, col in c.custom]
    return vk, custom


def _host_vk(pb, n, vk, custom):
    fq = lambda p: (pb.FQ(p[0]), pb.FQ(p[1]))  # noqa: E731
    base = [fq(vk[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")]
    return base, pb.g2_mul(pb.G2, TAU), pb.Scalar.root_of_unity(n), tuple((e, fq(p)) for e, p in custom)


# ---- CPU: exponents ------------------------------------------------------------------------------------------------
def test_three_exponent_terms_equal_their_padded_form(host_lincomb):
    pb = host_lincomb
    from plonkathon_b200.custom_gates import check_exponents, is_next_row, monomial, padded
    for e in [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]:
        six = e + (0, 0, 0)
        assert check_exponents([six]) == (six,) and padded(e) == six and not is_next_row(six)
        assert monomial(e, 3, 5, 7) == monomial(six, 3, 5, 7, 11, 13, 17)
        with pytest.raises(ValueError, match="twice"):
            check_exponents([e, six])
    # a plain custom-gate proof verifies under a key whose terms are written with six exponents
    c = syn.build_circuit(4, seed=21, n_public=2, custom=[(2, 0, 0), (1, 1, 1)])
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    proof = XO.prove(F.Setup(TAU, n), pk, A, B, C, c.public_values(), fast=True)
    vk, custom = _oracle_vk(c, pk)
    base, x2, w, terms = _host_vk(pb, n, vk, custom)
    key = pb.VerificationKey(n, *base, x2, w, tuple((e + (0, 0, 0), p) for e, p in terms))
    pf = pb.Proof.from_bytes(O.proof_bytes(proof))
    assert not key.next_row
    assert key.verify_proof(n, pf, c.public_values()) and key.verify_proof_unoptimized(n, pf, c.public_values())


@pytest.mark.parametrize("terms,match", [
    ([(0, 0, 0, 0, 0, 0)], "degree"), ([(0, 0, 0, 4, 0, 0)], "degree"), ([(1, 0, 0, 0, 3, 0)], "degree"),
    ([(1, 0, 0, 0, 0, 0)], "degree"), ([(0, 0, 1, 0, 0, 0)], "degree"), ([(1, 1, 0, 0, 0, 0)], "QM"),
    ([(0, 0, 0, 1, 0, 0), (0, 0, 0, 1, 0, 0)], "twice"), ([(1, 0, 0, 0, -1, 0)], "non-negative"),
    ([(0, 0, 0, 1)], "three"), ([(0, 0, 0, 1, 0, 0), (0, 0, 0, 0, 1, 0), (0, 0, 0, 0, 0, 1), (2, 0, 0), (0, 2, 0)],
                                "at most 4"),
])
def test_malformed_next_row_terms_are_rejected(terms, match):
    import plonkathon_b200 as pb
    n = 16
    pk = {k: np.zeros((n, 32), np.uint8) for k in PK_KEYS}
    custom = [(e, np.zeros((n, 32), np.uint8)) for e in terms]
    with pytest.raises(ValueError, match=match):
        pb.Prover.from_arrays(None, n, pk, custom=custom)
    with pytest.raises(ValueError, match=match):
        pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, custom=custom)
    with pytest.raises(ValueError, match=match):
        syn.build_circuit(4, custom=terms)


@pytest.mark.parametrize("e", [(0, 0, 0, 1, 0, 0), (0, 0, 0, 0, 1, 0), (0, 0, 0, 0, 0, 1)])
def test_next_row_degree_one_term_is_accepted(e):
    from plonkathon_b200.custom_gates import check_exponents, is_next_row
    assert check_exponents([e]) == (e,) and is_next_row(e)
    c = _circuit(4, 2, [e], 3)
    assert c.custom[0][0] == e


def test_next_row_terms_refused_with_lookups_and_on_the_sharded_prover():
    import plonkathon_b200 as pb
    from plonkathon_b200 import parallel
    n = 16
    pk = {k: np.zeros((n, 32), np.uint8) for k in PK_KEYS}
    custom = [((0, 0, 0, 1, 0, 0), np.zeros((n, 32), np.uint8))]
    table = ([1], [2], [3])
    qk = [0] * n
    for kw in ({"lookup": (qk, table)}, {"lookups": [(qk, table)]}):
        with pytest.raises(ValueError, match="next-row"):
            pb.Prover.from_arrays(None, n, pk, custom=custom, **kw)
        with pytest.raises(ValueError, match="next-row"):
            pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, custom=custom, **kw)
        with pytest.raises(ValueError, match="next-row"):
            syn.build_circuit(4, custom=[(0, 0, 0, 1, 0, 0)], **({"lookup": table} if "lookup" in kw else
                                                                 {"lookups": [table]}))
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.from_arrays(None, n, pk, custom=custom)


def test_plain_circuits_are_unchanged_by_the_next_row_builder():
    """build_circuit draws the same numbers for same-row terms however they are written"""
    a = syn.build_circuit(8, seed=77, n_public=2, custom=[(2, 0, 0), (1, 1, 1)])
    b = syn.build_circuit(8, seed=77, n_public=2, custom=[(2, 0, 0, 0, 0, 0), (1, 1, 1, 0, 0, 0)])
    assert a.values == b.values and a.QC == b.QC and np.array_equal(a.wire_L, b.wire_L)
    assert [col for _, col in a.custom] == [col for _, col in b.custom]


# ---- CPU: the oracle -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_next_row_proof_verifies(terms, log_n, host_lincomb):
    pb = host_lincomb
    c = _circuit(log_n, 2, terms, 100 + log_n)
    n = c.group_order
    pk, _, proof = _oracle_proof(c, fast=log_n > 4)  # 2^4: the pure-Python transforms
    vk, custom = _oracle_vk(c, pk)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=custom), proof, public, TAU)
    assert not XO.verify_proof_trapdoor(n, dict(vk, custom=custom), proof, [public[0] + 1] + public[1:], TAU)
    base, x2, w, terms_pt = _host_vk(pb, n, vk, custom)
    key = pb.VerificationKey(n, *base, x2, w, terms_pt)
    raw = XO.proof_bytes(proof)
    pf = pb.NextRowProof.from_bytes(raw)
    assert pf.to_bytes() == raw and key.next_row
    assert key.verify_proof(n, pf, public) and key.verify_proof_unoptimized(n, pf, public)


def test_oracle_running_sum_range_check_verifies(host_lincomb):
    pb = host_lincomb
    c = syn.range_check_circuit(6, 3, bits=16, seed=4)
    n = c.group_order
    pk, _, proof = _oracle_proof(c)
    vk, custom = _oracle_vk(c, pk)
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=custom), proof, [], TAU)
    base, x2, w, terms = _host_vk(pb, n, vk, custom)
    key = pb.VerificationKey(n, *base, x2, w, terms)
    pf = pb.NextRowProof.from_bytes(XO.proof_bytes(proof))
    assert key.verify_proof(n, pf, []) and key.verify_proof_unoptimized(n, pf, [])
    # a value that is not a running sum of bits: acc_1 = 2 breaks the first row of the first value
    A, B, C = c.wires_values()
    A[3] = 2
    with pytest.raises(AssertionError, match="gate 2 unsatisfied"):
        XO.prove(F.Setup(TAU, n), pk, A, B, C, [], fast=True)


def test_both_routines_reject_tampered_proofs_and_wrong_keys(host_lincomb):
    pb = host_lincomb
    c = _circuit(4, 2, ALL_TERMS, 21)
    n = c.group_order
    pk, _, proof = _oracle_proof(c)
    vk, custom = _oracle_vk(c, pk)
    base, x2, w, terms = _host_vk(pb, n, vk, custom)
    good = pb.VerificationKey(n, *base, x2, w, terms)
    public = c.public_values()
    raw = XO.proof_bytes(proof)
    pf = pb.NextRowProof.from_bytes(raw)
    assert good.verify_proof(n, pf, public) and good.verify_proof_unoptimized(n, pf, public)
    bad = {}
    for k in XO.FIELDS["next_row"]["4"]:
        bad["tampered " + k] = pb.NextRowProof.from_bytes(XO.proof_bytes(dict(proof, **{k: (proof[k] + 1) % R})))
    bad["swapped openings"] = pb.NextRowProof.from_bytes(
        XO.proof_bytes(dict(proof, W_z_1=proof["W_zw_1"], W_zw_1=proof["W_z_1"])))
    bad["a plain proof"] = pb.Proof.from_bytes(raw[:768])
    for why, p in bad.items():
        assert not good.verify_proof(n, p, public), why
        assert not good.verify_proof_unoptimized(n, p, public), why
    # a key whose next-row exponents are relabelled to the same row (the other terms keep the key a next-row key)
    relabel = {(0, 0, 0, 0, 2, 1): (0, 2, 1, 0, 0, 0), (0, 1, 1, 0, 0, 1): (0, 1, 2, 0, 0, 0)}
    for old, new in relabel.items():
        t = tuple((new if e == old else e, p) for e, p in terms)
        key = pb.VerificationKey(n, *base, x2, w, t)
        assert key.next_row
        assert not key.verify_proof(n, pf, public), (old, new)
        assert not key.verify_proof_unoptimized(n, pf, public), (old, new)
    # and a plain key refuses a next-row proof
    plain = pb.VerificationKey(n, *base, x2, w)
    assert not plain.verify_proof(n, pf, public) and not plain.verify_proof_unoptimized(n, pf, public)


def test_non_canonical_next_row_encoding_is_rejected():
    import plonkathon_b200 as pb
    c = _circuit(4, 2, ALL_TERMS, 21)
    _, _, proof = _oracle_proof(c)
    raw = XO.proof_bytes(proof)
    for word in (24, 25, 26):
        x = int.from_bytes(raw[32 * word:32 * word + 32], "big") + R
        with pytest.raises(ValueError, match="word %d" % word):
            pb.NextRowProof.from_bytes(raw[:32 * word] + x.to_bytes(32, "big") + raw[32 * word + 32:])
    with pytest.raises(ValueError, match="864"):
        pb.NextRowProof.from_bytes(raw[:768])


def _wrapping_circuit(log_n, seed):
    """a full circuit whose last row carries a term over a(wX): it reads row 0"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=2, custom=[(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0)])
        n = c.group_order
        if c.n_constraints == n and any(col[n - 1] for _, col in c.custom):
            return c
        seed += 1


def test_oracle_rejects_a_broken_wrap_around_row():
    c = _wrapping_circuit(5, 1)
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    public = c.public_values()
    XO.prove(F.Setup(TAU, n), pk, A, B, C, public, fast=True)  # the witness as built proves
    # row 0 is a public row: moving its value and the public input together keeps row 0 and breaks row n - 1
    A[0], public = (A[0] + 1) % R, [(public[0] + 1) % R] + public[1:]
    with pytest.raises(AssertionError, match="gate %d unsatisfied" % (n - 1)):
        XO.prove(F.Setup(TAU, n), pk, A, B, C, public, fast=True)


def test_oracle_zk_proof_verifies_and_blinded_wires_agree_on_h(host_lincomb):
    pb = host_lincomb
    c = _circuit(5, 2, ALL_TERMS, 40)
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n + 9)
    with F.c_kernels():
        prover = XO.Prover(setup, pk, _blinders(5))
        proof = prover.prove(A, B, C, c.public_values())
        plain = XO.prove(setup, pk, A, B, C, c.public_values())
    roots = O.roots_of_unity(n)
    for blinded, vals in ((prover.Ab, A), (prover.Bb, B), (prover.Cb, C)):
        assert len(blinded) == n + 3 and any(blinded[n:])
        assert [XO.poly_eval(blinded, x) for x in roots] == [v % R for v in vals]
    vk, custom = _oracle_vk(c, pk)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=custom), proof, public, TAU)
    base, x2, w, terms = _host_vk(pb, n, vk, custom)
    key = pb.VerificationKey(n, *base, x2, w, terms)
    pf = pb.NextRowProof.from_bytes(XO.proof_bytes(proof))
    assert key.verify_proof(n, pf, public) and key.verify_proof_unoptimized(n, pf, public)
    assert proof["a_1"] != plain["a_1"] and proof["a_shifted_eval"] != plain["a_shifted_eval"]
    # zero blinders give the plain next-row proof
    with F.c_kernels():
        zero = XO.Prover(setup, pk, [0] * 14).prove(A, B, C, public)
    assert XO.proof_bytes(zero) == XO.proof_bytes(plain)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _gpu_prover(pb, c, setup=None, extra=0):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n + extra)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c))
    return setup, pk, prover, (A, B, C, public)


GPU_SIZES = [(4, 2), (8, 2), (12, 2), (8, 11), (12, 9)]


@pytest.mark.gpu
@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n,n_public", GPU_SIZES)
def test_gpu_next_row_proof_equals_oracle(terms, log_n, n_public):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated (the two paths of k_quotient)"""
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, terms, 200 + log_n + n_public)
    _, _, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    assert len(raw) == 864 and prover.next_row
    _, _, proof = _oracle_proof(c)
    assert raw == XO.proof_bytes(proof)


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [ALL_TERMS, list(syn.RUNNING_SUM_TERMS)], ids=["all4", "running_sum"])
@pytest.mark.parametrize("log_n,n_public", GPU_SIZES)
def test_gpu_zk_next_row_proof_equals_oracle(terms, log_n, n_public):
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, terms, 300 + log_n + n_public)
    _, _, prover, wires = _gpu_prover(pb, c, extra=9)
    blinders = _blinders(log_n + n_public)
    prover.set_zk(True, blinders)
    raw = prover.prove_arrays(*wires)
    _, _, proof = _oracle_proof(c, blinders=blinders)
    assert raw == XO.proof_bytes(proof)


@pytest.mark.gpu
@pytest.mark.parametrize("zk", [False, True], ids=["plain", "zk"])
def test_gpu_round_by_round_abi_gives_the_whole_proof(zk):
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    from plonkathon_b200.transcript import NextRowMessage4, Transcript
    c = _circuit(8, 2, ALL_TERMS, 55)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c, extra=9)
    if zk:
        prover.set_zk(True, _blinders(8))
    whole = prover.prove_arrays(A, B, C, public)
    tr = Transcript(b"plonk")
    msg_1 = prover.round_1_arrays(A, B, C, public)
    prover.beta, prover.gamma = tr.round_1(msg_1)
    msg_2 = prover.round_2()
    prover.alpha, prover.fft_cofactor = tr.round_2(msg_2)
    msg_3 = prover.round_3()
    prover.zeta = tr.round_3(msg_3)
    msg_4 = prover.round_4()
    assert isinstance(msg_4, NextRowMessage4)
    prover.v = tr.round_4(msg_4)
    msg_5 = prover.round_5()
    m4 = pb.prover.Message4(*[getattr(msg_4, k) for k in pb.prover.PROOF_FIELDS[7:13]])
    pf = pb.NextRowProof(pb.Proof(msg_1, msg_2, msg_3, m4, msg_5), msg_4.a_shifted_eval, msg_4.b_shifted_eval,
                         msg_4.c_shifted_eval)
    assert pf.to_bytes() == whole
    out = ctypes.create_string_buffer(864)
    _lib.check(_lib.lib().pb200_prover_serialize_next_row(prover._h, out))
    assert out.raw == whole


@pytest.mark.gpu
def test_gpu_golden_next_row_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_next_row_2p16.json")))
    c = syn.range_check_circuit(rec["log_n"], rec["n_values"], bits=rec["bits"], seed=rec["seed"])
    assert [list(e) for e, _ in c.custom] == rec["terms"]
    n = c.group_order
    setup, pk, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden next-row proof"
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c))
    assert [(e, (p[0].n, p[1].n)) for e, p in vk.custom] == [(tuple(e), pt(p)) for e, p in rec["vk_custom"]]
    public = [int(x) for x in rec["public"]]
    pf = pb.NextRowProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_fresh_blinders_differ_and_verify():
    import plonkathon_b200 as pb
    c = _circuit(10, 2, ALL_TERMS, 61)
    n = c.group_order
    setup, pk, prover, wires = _gpu_prover(pb, c, extra=9)
    prover.set_zk(True)
    p1, p2 = prover.prove_arrays(*wires), prover.prove_arrays(*wires)
    assert p1 != p2
    f1, f2 = pb.NextRowProof.from_bytes(p1).flatten(), pb.NextRowProof.from_bytes(p2).flatten()
    changed = [k for k in f1 if f1[k] != f2[k]]
    # every commitment but none of S1, S2 at zeta (the challenges differ, so those change too): all 18 fields move
    assert len(changed) == len(f1), changed
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c))
    public = c.public_values()
    for raw in (p1, p2):
        pf = pb.NextRowProof.from_bytes(raw)
        assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_next_row_2p20_verifies():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, custom=ALL_TERMS)
    n = c.group_order
    setup, pk, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c))
    public = c.public_values()
    pf = pb.NextRowProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    k = 768  # a_shifted_eval
    bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not vk.verify_proof(n, pb.NextRowProof.from_bytes(bad), public)
    assert not vk.verify_proof_unoptimized(n, pb.NextRowProof.from_bytes(bad), public)


@pytest.mark.gpu
def test_gpu_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, parallel
    L = _lib.lib()
    c = _circuit(8, 2, ALL_TERMS, 71)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c, extra=9)
    prover.prove_arrays(A, B, C, public)
    err = lambda: L.pb200_last_error().decode()  # noqa: E731
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    pub = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in public), np.uint8).reshape(-1, 32).copy()
    out = ctypes.create_string_buffer(1216)
    # the 768-byte entry points
    assert L.pb200_prover_prove(prover._h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out) != 0
    assert "864 bytes" in err() and "pb200_prover_prove_next_row" in err()
    assert L.pb200_prover_serialize(prover._h, out) != 0 and "864 bytes" in err()
    assert L.pb200_prover_round4(prover._h, bytes(32), out) != 0 and "pb200_prover_round4_next_row" in err()
    import torch
    d = [torch.from_numpy(x).cuda() for x in (A, B, C)]
    assert L.pb200_prover_prove_device(prover._h, *[ctypes.c_void_p(t.data_ptr()) for t in d], ptr(pub), len(public),
                                       out) != 0
    assert "864 bytes" in err()
    # lookups
    with pytest.raises(_lib.PlonkB200Error, match="next-row"):
        prover._set_lookup([0] * n, ([1], [2], [3]), 1)
    # the next-row entry points on a plain prover
    plain = pb.Prover.from_arrays(setup, n, pk, custom=[((2, 0, 0), np.zeros((n, 32), np.uint8))])
    assert not plain.next_row
    assert L.pb200_prover_prove_next_row(plain._h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out) != 0
    assert "no next-row" in err()
    # sharded creation
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.from_arrays(setup, n, pk, custom=syn.custom_arrays(c))
    # zero knowledge: 14 blinders, an SRS of n + 9 powers, n >= 16
    with pytest.raises(ValueError, match="14 blinders"):
        prover.set_zk(True, [1] * 11)
    short = pb.Prover.from_arrays(pb.Setup.generate(TAU, n + 8), n, pk, custom=syn.custom_arrays(c))
    with pytest.raises(_lib.PlonkB200Error, match=r"n \+ 9 powers"):
        short.set_zk(True)
    c8 = syn.build_circuit(3, seed=1, n_public=1, custom=[(0, 0, 0, 1, 0, 0)])
    _, _, small, _ = _gpu_prover(pb, c8, extra=9)
    with pytest.raises(_lib.PlonkB200Error, match="n >= 16"):
        small.set_zk(True)
    # a refused call left the provers usable
    assert prover.prove_arrays(A, B, C, public) == prover.prove_arrays(A, B, C, public)


@pytest.mark.gpu
def test_gpu_broken_wrap_around_row_raises():
    import plonkathon_b200 as pb
    c = _wrapping_circuit(10, 1)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c)
    bad = A.copy()
    bad[0] = np.frombuffer(((int.from_bytes(A[0].tobytes(), "little") + 1) % R).to_bytes(32, "little"), np.uint8)
    bad_public = [(public[0] + 1) % R] + public[1:]
    with pytest.raises(AssertionError, match="gate constraints"):
        prover.prove_arrays(bad, B, C, bad_public)
    assert prover.prove_arrays(A, B, C, public)


@pytest.mark.gpu
def test_gpu_same_row_six_exponent_terms_take_the_plain_path():
    """terms written with six exponents and no next-row one give the 768-byte custom-gate proof"""
    import plonkathon_b200 as pb
    terms = [(2, 0, 0), (1, 1, 1)]
    c = syn.build_circuit(8, seed=31, n_public=2, custom=terms)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    three = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c))
    six = pb.Prover.from_arrays(setup, n, pk, custom=[(e + (0, 0, 0), col) for e, col in syn.custom_arrays(c)])
    assert not six.next_row
    raw = six.prove_arrays(A, B, C, public)
    assert len(raw) == 768 and raw == three.prove_arrays(A, B, C, public)
    proof = XO.prove(F.Setup(TAU, n), XO.preprocessed(c), *c.wires_values(), public, fast=True)
    assert raw == O.proof_bytes(proof)
