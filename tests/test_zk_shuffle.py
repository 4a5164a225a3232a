"""Zero-knowledge shuffle proofs: the blinding of zero-knowledge mode plus Z3 (tests/extended_oracle.py has the
construction), with the 896- and 992-byte proofs, the transcript and the verifier unchanged.

CPU: with zero blinders the oracle gives the bytes of the shuffle proofs tests/golden/oracle_kinds.json pins for plain, same-row
and next-row circuits; with random blinders its proofs pass the trapdoor check and both host verifier routines, and
tampered ones do not; Z3' agrees with Z3 on H and the blinded quotient pieces recombine to T; the z3_1 a witness guess
recomputes from the transcript's theta and kappa matches a plain shuffle proof and no zero-knowledge one; the Python
argument checks of ``set_zk_shuffle``.  GPU: the prover's bytes equal the oracle's with fixed blinders, zero blinders
reproduce the shuffle golden, the 2^16 zero-knowledge shuffle golden is reproduced, fresh blinders change every
commitment and every blinded evaluation and verify, the round-by-round path gives the whole proof, the mode switches off
through either entry point, the refusals leave the prover usable, and a 2^20 proof verifies."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest

from oracle import fast as F
from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from tests import extended_oracle as XO
from tests.golden.make_oracle_kinds import circuit, pinned
from tests.oracle_keys import host_lincomb  # noqa: F401  (a fixture)
from tests.golden_io import GOLDEN
from tests.test_shuffle import (GPU_SIZES, GPU_TERM_IDS, GPU_TERMS, NEXT_TERMS, TERM_IDS, TERM_SETS, _circuit, _host_key,
                                _host_proof, _oracle_vk, _skewed_circuit)

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
POINTS = ("a_1", "b_1", "c_1", "z_1", "t_lo_1", "t_mid_1", "t_hi_1", "W_z_1", "W_zw_1", "z3_1")


def _blinders(count, seed):
    rng = random.Random(seed)
    return [rng.randrange(1, R) for _ in range(count)]


def _oracle(c, blinders, fast=True):
    """(pk, proof, prover object) of the zero-knowledge oracle on an SRS of n + 9 powers"""
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n + 9)
    if not fast:
        setup = O.Setup([setup.point(i) for i in range(n + 9)], None)
    prover = XO.Prover(setup, pk, blinders)
    if fast:
        with F.c_kernels():
            proof = prover.prove(A, B, C, c.public_values())
    else:
        proof = prover.prove(A, B, C, c.public_values())
    return pk, proof, prover


# ---- CPU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_zero_blinders_give_the_shuffle_proof(terms, log_n):
    """against the shuffle proofs that tests/golden/oracle_kinds.json pins"""
    rec = pinned("shuffle", log_n, terms)
    c = circuit(rec)
    _, proof, _ = _oracle(c, [0] * XO.blinder_count(XO.preprocessed(c)), fast=log_n > 4)
    assert hashlib.sha256(XO.proof_bytes(proof)).hexdigest() == rec["sha256"]


@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_zk_shuffle_proof_verifies(terms, log_n, host_lincomb):
    pb = host_lincomb
    c = _circuit(log_n, 2, terms, 200 + log_n)
    n = c.group_order
    pk = XO.preprocessed(c)
    _, proof, _ = _oracle(c, _blinders(XO.blinder_count(pk), log_n), fast=log_n > 4)
    vk, custom, shuffle = _oracle_vk(c, pk)
    public = c.public_values()
    key = _host_key(pb, n, vk, custom, shuffle)
    bad = [dict(proof, **{k: (proof[k] + 1) % R}) for k in ("z3_shifted_eval", "a_eval")]
    bad.append(dict(proof, W_z_1=proof["W_zw_1"], W_zw_1=proof["W_z_1"]))
    for p, ok in [(proof, True)] + [(b, False) for b in bad]:
        assert XO.verify_proof_trapdoor(n, dict(vk, custom=custom, shuffle=shuffle), p, public, TAU) is ok
        if log_n == 8 and not ok:
            continue  # the host routines' rejections once per term set, at the smaller sizes
        raw = XO.proof_bytes(p)
        assert len(raw) == (992 if terms == NEXT_TERMS else 896)
        pf = _host_proof(pb, raw)
        assert key.verify_proof(n, pf, public) is ok and key.verify_proof_unoptimized(n, pf, public) is ok


@pytest.mark.parametrize("terms", [[], NEXT_TERMS], ids=["plain", "next_row"])
def test_oracle_blinded_z3_agrees_on_h_and_pieces_recombine(terms):
    c = _circuit(6, 2, terms, 17)
    n = c.group_order
    pk = XO.preprocessed(c)
    _, _, prover = _oracle(c, _blinders(XO.blinder_count(pk), 5))
    w = O.root_of_unity(n)
    assert len(prover.Z3c) == n + 3 and prover.Z3c[n:] != [0, 0, 0]
    assert [XO.poly_eval(prover.Z3c, pow(w, i, R)) for i in range(n)] == prover.Z3
    T = prover.T
    assert any(T[3 * n:])  # the blinded quotient reaches past 3n
    assert not any(T[3 * n + (9 if terms else 6):])  # deg T <= 3n + 5 (3n + 8 with next-row terms)
    x = random.Random(7).randrange(R)
    xn = pow(x, n, R)
    got = (XO.poly_eval(prover.T1b, x) + xn * XO.poly_eval(prover.T2b, x) + xn * xn * XO.poly_eval(prover.T3b, x)) % R
    assert got == XO.poly_eval(T, x)


def _guess_z3_1(c, proof):
    """z3_1 recomputed from the witness and the theta, kappa of the proof's own transcript"""
    n = c.group_order
    ch = XO.challenges(proof)
    th, ka = ch["theta"], ch["kappa"]
    A, B, C = ([int(v) % R for v in X] for X in c.wires_values())
    q_in, q_out = c.shuffle
    Z3 = [1]
    for i in range(n - 1):
        t = (ka + A[i] + th * B[i] + th * th % R * C[i]) % R
        Z3.append(Z3[-1] * (t if q_in[i] else 1) % R * O.inv0(t if q_out[i] else 1, R) % R)
    with F.c_kernels():
        return F.Setup(TAU, n).commit(Z3)


@pytest.mark.parametrize("terms", [[], NEXT_TERMS], ids=["plain", "next_row"])
def test_witness_guess_matches_plain_shuffle_proofs_only(terms):
    """whoever knows the witness recomputes Z3 and its commitment from the public theta, kappa: equal to a plain shuffle
    proof's z3_1 (the test can see the leak), different from every zero-knowledge shuffle proof's"""
    c = _circuit(6, 2, terms, 300)
    n = c.group_order
    pk = XO.preprocessed(c)
    plain = XO.prove(F.Setup(TAU, n), pk, *c.wires_values(), c.public_values(), fast=True)
    assert _guess_z3_1(c, plain) == plain["z3_1"]
    for seed in (1, 2):
        _, zk, _ = _oracle(c, _blinders(XO.blinder_count(pk), seed))
        assert _guess_z3_1(c, zk) != zk["z3_1"]


def test_set_zk_shuffle_argument_checks():
    import plonkathon_b200 as pb
    from plonkathon_b200 import parallel
    p = pb.Prover.__new__(pb.Prover)
    with pytest.raises(ValueError, match="14 blinders"):
        p.set_zk_shuffle(True, [1] * 11)
    with pytest.raises(ValueError, match=r"\[0, r\)"):
        p.set_zk_shuffle(True, [1] * 13 + [R])
    p.next_row = True
    with pytest.raises(ValueError, match="17 blinders"):
        p.set_zk_shuffle(True, [1] * 14)
    with pytest.raises(ValueError, match=r"\[0, r\)"):
        p.set_zk_shuffle(True, [-1] + [1] * 16)
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.__new__(parallel.ShardedProver).set_zk_shuffle(True)


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _gpu_prover(pb, c, setup=None, blinders=None, zk=True):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n + 9)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))
    if zk:
        prover.set_zk_shuffle(True, blinders)
    return setup, pk, prover, (A, B, C, public)


def _vk(setup, c, pk):
    return setup.verification_key_arrays(c.group_order, pk, custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))


def _count(c):
    return XO.blinder_count(XO.preprocessed(c))


@pytest.mark.gpu
@pytest.mark.parametrize("terms", GPU_TERMS, ids=GPU_TERM_IDS)
@pytest.mark.parametrize("log_n,n_public", GPU_SIZES)
def test_gpu_zk_shuffle_proof_equals_oracle(terms, log_n, n_public):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated"""
    import plonkathon_b200 as pb
    seed = 500 + log_n + n_public
    c = _circuit(log_n, n_public, terms, seed)
    bl = _blinders(_count(c), seed)
    _, _, prover, wires = _gpu_prover(pb, c, blinders=bl)
    raw = prover.prove_arrays(*wires)
    _, proof, _ = _oracle(c, bl)
    assert len(raw) == (896 if terms in ([], [(2, 0, 0), (1, 1, 1)]) else 992)
    assert raw == XO.proof_bytes(proof)
    assert prover.prove_arrays(*wires) == raw  # fixed blinders: the same proof again


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [4, 8, 12])
def test_gpu_skewed_zk_shuffle_equals_oracle(log_n):
    import plonkathon_b200 as pb
    c = _skewed_circuit(log_n)
    bl = _blinders(14, log_n)
    _, _, prover, wires = _gpu_prover(pb, c, blinders=bl)
    raw = prover.prove_arrays(*wires)
    _, proof, _ = _oracle(c, bl)
    assert len(raw) == 896 and raw == XO.proof_bytes(proof)


def _golden_circuit(rec):
    return syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                             custom=[tuple(e) for e in rec["terms"]], shuffle=True)


@pytest.mark.gpu
def test_gpu_zero_blinders_reproduce_the_shuffle_golden():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_shuffle_2p16.json")))
    c = _golden_circuit(rec)
    setup = pb.Setup.generate(TAU, c.group_order + 9)
    _, _, prover, wires = _gpu_prover(pb, c, setup, [0] * 17)
    assert prover.prove_arrays(*wires).hex() == rec["proof_hex"]


@pytest.mark.gpu
def test_gpu_golden_zk_shuffle_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_zk_shuffle_2p16.json")))
    c = _golden_circuit(rec)
    n = c.group_order
    assert sum(c.shuffle[0]) == rec["rows_in"]
    setup = pb.Setup.generate(TAU, rec["srs_powers"])
    _, pk, prover, wires = _gpu_prover(pb, c, setup, [int(b) for b in rec["blinders"]])
    raw = prover.prove_arrays(*wires)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden zero-knowledge shuffle proof"
    vk = _vk(setup, c, pk)
    pf = pb.NextRowShuffleProof.from_bytes(raw)
    pub = [int(x) for x in rec["public"]]
    assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)


def _proof_dict(pb, raw):
    """a proof's fields as the oracle's dict: points as (x, y) ints, scalars as ints"""
    return {k: (int(v[0].n), int(v[1].n)) if isinstance(v, tuple) else int(v.n)
            for k, v in _host_proof(pb, raw).flatten().items()}


def _tamper_word(raw, k):
    """raw with 32-byte word k (counted from the start of the proof) incremented"""
    x = (int.from_bytes(raw[32 * k:32 * k + 32], "big") + 1) % R
    return raw[:32 * k] + x.to_bytes(32, "big") + raw[32 * k + 32:]


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [[], NEXT_TERMS], ids=["plain", "next_row"])
def test_gpu_fresh_blinders_differ_and_verify(terms):
    import plonkathon_b200 as pb
    c = _circuit(10, 2, terms, 12)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c)
    p1 = prover.prove_arrays(A, B, C, public)
    p2 = prover.prove_arrays(A, B, C, public)
    f1, f2 = (_proof_dict(pb, raw) for raw in (p1, p2))
    blinded = ["a_eval", "b_eval", "c_eval", "z_shifted_eval", "z3_shifted_eval"]
    if terms:
        blinded += ["a_shifted_eval", "b_shifted_eval", "c_shifted_eval"]
    assert all(f1[k] != f2[k] for k in POINTS + tuple(blinded))
    # zeta differs between the two proofs, so no evaluation repeats; the fixed polynomials S1, S2 and Q_in are not
    # blinded, so their evaluations are those of the columns at each proof's own zeta, and the wires' are not
    spk = XO.preprocessed(c)
    A_ = [int(v) % R for v in c.wires_values()[0]]
    for f in (f1, f2):
        zeta = XO.challenges(f)["zeta"]
        for k, col in (("s1_eval", spk.S1), ("s2_eval", spk.S2), ("qin_eval", spk.q_in)):
            assert f[k] == O.barycentric_eval(col, zeta), k
        assert f["a_eval"] != O.barycentric_eval(A_, zeta)
    vk = _vk(setup, c, pk)
    for raw in (p1, p2):
        pf = _host_proof(pb, raw)
        assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [[], NEXT_TERMS], ids=["plain", "next_row"])
def test_gpu_round_by_round_abi_gives_the_whole_proof(terms):
    """fixed blinders: the rounds through the C ABI, fed the challenges of the whole proof's transcript, give its bytes"""
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    c = _circuit(8, 2, terms, 55)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c, blinders=_blinders(_count(c), 55))
    raw = prover.prove_arrays(A, B, C, public)
    ch = XO.challenges(_proof_dict(pb, raw))
    le = lambda k: (int(ch[k]) % R).to_bytes(32, "little")  # noqa: E731
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    pub = np.ascontiguousarray(np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in public), np.uint8))
    L, h, out = _lib.lib(), prover._h, ctypes.create_string_buffer(992)
    _lib.check(L.pb200_prover_round1(h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out))
    _lib.check(L.pb200_prover_round2_shuffle(h, le("beta"), le("gamma"), le("theta"), le("kappa"), out))
    _lib.check(L.pb200_prover_round3(h, le("alpha"), le("fft_cofactor"), out))
    r4 = L.pb200_prover_round4_next_row_shuffle if terms else L.pb200_prover_round4_shuffle
    _lib.check(r4(h, le("zeta"), out))
    _lib.check(L.pb200_prover_round5(h, le("v"), out))
    ser = L.pb200_prover_serialize_next_row_shuffle if terms else L.pb200_prover_serialize_shuffle
    _lib.check(ser(h, out))
    assert out.raw[:len(raw)] == raw


@pytest.mark.gpu
def test_gpu_switching_and_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, parallel
    rec = json.load(open(os.path.join(GOLDEN, "proof_shuffle_2p16.json")))
    c = _golden_circuit(rec)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c, pb.Setup.generate(TAU, n + 9), zk=False)
    vk = _vk(setup, c, pk)
    golden = lambda: prover.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]  # noqa: E731
    assert golden()
    for off in (lambda: prover.set_zk_shuffle(False), lambda: prover.set_zk(False)):
        prover.set_zk_shuffle(True)
        raw = prover.prove_arrays(A, B, C, public)
        assert raw.hex() != rec["proof_hex"]
        assert vk.verify_proof(n, pb.NextRowShuffleProof.from_bytes(raw), public)
        with pytest.raises(RuntimeError, match="T1"):
            prover.T1
        off()
        assert not prover.zk and golden()
    # refusals, each leaving the prover as it was
    L = _lib.lib()
    assert L.pb200_prover_set_zk_shuffle(prover._h, 1, b"\xff" * 32 * 17) != 0
    assert "not reduced" in L.pb200_last_error().decode()
    with pytest.raises(_lib.PlonkB200Error, match="does not combine with a shuffle"):
        prover.set_zk(True)
    assert golden()
    prover.set_zk_shuffle(True, [0] * 17)
    with pytest.raises(_lib.PlonkB200Error, match="does not combine with a shuffle"):
        prover.set_zk(True, [0] * 14)
    assert golden()  # still in zero-knowledge shuffle mode, with zero blinders
    prover.set_zk_shuffle(False)
    plain = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c))
    with pytest.raises(_lib.PlonkB200Error, match="no shuffle"):
        plain.set_zk_shuffle(True)
    plain.set_zk(True)
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge"):
        plain._set_shuffle(*syn.shuffle_arrays(c))
    assert len(plain.prove_arrays(A, B, C, public)) == 864
    short = pb.Prover.from_arrays(pb.Setup.generate(TAU, n + 6), n, pk, custom=syn.custom_arrays(c),
                                  shuffle=syn.shuffle_arrays(c))
    with pytest.raises(_lib.PlonkB200Error, match=r"n \+ 9"):
        short.set_zk_shuffle(True)
    assert short.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]
    small = _circuit(3, 0, NEXT_TERMS, 3)  # n = 8: next-row terms need n >= 16
    _, _, sp, _ = _gpu_prover(pb, small, pb.Setup.generate(TAU, 64), zk=False)
    with pytest.raises(_lib.PlonkB200Error, match="n >= 16"):
        sp.set_zk_shuffle(True)
    tiny = _circuit(2, 0, [], 3)  # n = 4
    _, _, tp, _ = _gpu_prover(pb, tiny, pb.Setup.generate(TAU, 64), zk=False)
    with pytest.raises(_lib.PlonkB200Error, match="n >= 8"):
        tp.set_zk_shuffle(True)
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.__new__(parallel.ShardedProver).set_zk_shuffle(True)
    assert golden()


@pytest.mark.gpu
def test_gpu_zk_shuffle_2p20_verifies():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, custom=NEXT_TERMS, shuffle=True)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c)
    raw = prover.prove_arrays(A, B, C, public)
    vk = _vk(setup, c, pk)
    pf = pb.NextRowShuffleProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    bad = pb.NextRowShuffleProof.from_bytes(_tamper_word(raw, 992 // 32 - 1))  # z3_shifted_eval
    assert not vk.verify_proof(n, bad, public) and not vk.verify_proof_unoptimized(n, bad, public)
