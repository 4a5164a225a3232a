"""Zero-knowledge lookup proofs: the blinding of plain zero-knowledge mode plus F, H1, H2 and Z2 (tests/extended_oracle.py
has the construction), with the 1216-byte proof, the transcript and the verifier unchanged.

CPU: with zero blinders the oracle gives the bytes of the lookup proofs tests/golden/oracle_kinds.json pins (one
table untagged, two and three tagged); with random blinders its proofs pass the trapdoor check and both host verifier
routines, and tampered ones do not; the blinded polynomials agree with the unblinded ones on H and the blinded quotient
pieces recombine to T; the lookup commitments a witness guess recomputes from the transcript's eta match a plain lookup
proof and none of a zero-knowledge one.  GPU: the prover's 1216 bytes equal the oracle's with fixed blinders, zero
blinders reproduce the lookup goldens, the 2^16 zero-knowledge lookup golden is reproduced, fresh blinders change every
commitment and verify, the round-by-round path gives the whole proof, the mode switches off through either entry point,
the refusals leave the prover usable, and a 2^20 proof verifies."""
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
from tests import test_lookup as TLK
from tests.golden.make_oracle_kinds import circuit, pinned
from tests.golden_io import GOLDEN
from tests.oracle_keys import host_lincomb  # noqa: F401  (a fixture)
from tests.test_lookup import _commit_col, _host_vk
from tests.test_lookup_tagged import _circuit as _tagged_circuit
from tests.test_lookup_tagged import and_table, range_table, tables, xor_table

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
TERM = [(2, 0, 0)]
POINTS = ("a_1", "b_1", "c_1", "z_1", "t_lo_1", "t_mid_1", "t_hi_1", "W_z_1", "W_zw_1", "f_1", "h1_1", "h2_1", "z2_1")


def _blinders(seed):
    rng = random.Random(seed)
    return [rng.randrange(1, R) for _ in range(21)]


def _circuit(log_n, n_public, count, custom, seed):
    """one table through ``lookup=`` (the range table of ``tables``), two or three through ``lookups=``"""
    n = 1 << log_n
    if count == 1:
        return TLK._circuit(log_n, n_public, tables(n, 3)[0], custom, seed)
    return _tagged_circuit(log_n, n_public, tables(n, count), custom, seed)


def _oracle(c, blinders, fast=True):
    """(pk, setup of n + 6 powers, proof, prover object)"""
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n + 6)
    prover = XO.Prover(setup, pk, blinders)
    if fast:
        with F.c_kernels():
            proof = prover.prove(A, B, C, c.public_values())
    else:
        proof = prover.prove(A, B, C, c.public_values())
    return pk, setup, proof, prover


def _plain_oracle(c, fast=True):
    """the lookup oracles' proof: untagged for ``lookup=``, tagged for ``lookups=``"""
    n = c.group_order
    A, B, C = c.wires_values()
    if c.lookups:
        return XO.prove(F.Setup(TAU, n), XO.preprocessed(c), A, B, C, c.public_values(), fast=fast)
    return XO.prove(F.Setup(TAU, n), XO.preprocessed(c), A, B, C, c.public_values(), fast=fast)


def _oracle_vk(c, pk, setup):
    vk = {k: _commit_col(setup, col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO),
                                                    ("Qc", c.QC), ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom = [(e, _commit_col(setup, col)) for e, col in c.custom]
    cols = [pk.qk] + pk.table + ([pk.qtag, pk.t4] if c.lookups else [])
    return vk, custom, tuple(_commit_col(setup, col) for col in cols)


# ---- CPU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count", [1, 2, 3])
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_zero_blinders_give_the_lookup_proof(log_n, count):
    """against the lookup proofs, one table untagged, that tests/golden/oracle_kinds.json pins"""
    rec = pinned("lookup", log_n, (), count)
    _, _, proof, _ = _oracle(circuit(rec), [0] * 21, fast=log_n > 4)
    assert hashlib.sha256(XO.proof_bytes(proof)).hexdigest() == rec["sha256"]


@pytest.mark.parametrize("custom", [(), TERM], ids=["plain", "x2"])
@pytest.mark.parametrize("count", [1, 2, 3])
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_zk_lookup_proof_verifies(log_n, count, custom, host_lincomb):
    pb = host_lincomb
    n = 1 << log_n
    c = _circuit(log_n, 2, count, custom, 200 + log_n + count)
    pk, setup, proof, _ = _oracle(c, _blinders(log_n + count), fast=log_n > 4)
    vk, cpts, lpts = _oracle_vk(c, pk, setup)
    public = c.public_values()
    key = _host_vk(pb, c, vk, cpts, lpts)
    bad = [dict(proof, **{k: (proof[k] + 1) % R}) for k in ("f_eval", "h1_shifted_eval", "z2_shifted_eval")]
    bad.append(dict(proof, W_z_1=proof["W_zw_1"], W_zw_1=proof["W_z_1"]))
    for p, ok in [(proof, True)] + [(b, False) for b in bad]:
        assert XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), p, public, TAU) is ok
        if log_n == 8 and not ok:
            continue  # the host routines' rejections once per table count and term, at the smaller sizes
        pf = pb.LookupProof.from_bytes(XO.proof_bytes(p))
        assert key.verify_proof(n, pf, public) is ok and key.verify_proof_unoptimized(n, pf, public) is ok


def test_oracle_blinded_polynomials_agree_on_h_and_pieces_recombine():
    c = _circuit(6, 2, 3, (), 17)
    n = c.group_order
    _, _, _, prover = _oracle(c, _blinders(5))
    w = O.root_of_unity(n)
    for name, blinded, length in (("F", prover.Fb, n + 2), ("H1", prover.H1b, n + 3), ("H2", prover.H2b, n + 2),
                                  ("Z2", prover.Z2b, n + 3)):
        assert len(blinded) == length and blinded[n:] != [0] * (length - n), name
        assert [XO.poly_eval(blinded, pow(w, i, R)) for i in range(n)] == getattr(prover, name), name
    assert any(prover.T[3 * n:])  # the blinded quotient reaches past 3n
    x = random.Random(7).randrange(R)
    xn = pow(x, n, R)
    got = (XO.poly_eval(prover.T1b, x) + xn * XO.poly_eval(prover.T2b, x) + xn * xn * XO.poly_eval(prover.T3b, x)) % R
    assert got == XO.poly_eval(prover.T, x)


def _guess_commitments(c, proof):
    """f_1, h1_1, h2_1 recomputed from the witness and the eta of the proof's own transcript"""
    n = c.group_order
    setup = F.Setup(TAU, n)
    guess = XO.Prover(setup, XO.preprocessed(c))
    guess.PI = [(-int(v)) % R for v in c.public_values()] + [0] * (n - len(c.public_values()))
    with F.c_kernels():
        guess.round_1(*c.wires_values())
        guess.eta = XO.challenges(proof)["eta"]
        return tuple(guess.round_1L().values())


@pytest.mark.parametrize("count", [1, 3])
def test_witness_guess_matches_plain_lookup_proofs_only(count):
    """whoever knows the witness recomputes F, H1, H2 and their commitments from the public eta: equal to a plain lookup
    proof's (the test can see the leak), different from a zero-knowledge lookup proof's"""
    c = _circuit(6, 2, count, (), 300 + count)
    plain = _plain_oracle(c)
    assert _guess_commitments(c, plain) == (plain["f_1"], plain["h1_1"], plain["h2_1"])
    _, _, zk, _ = _oracle(c, _blinders(count))
    guess = _guess_commitments(c, zk)
    assert all(g != zk[k] for g, k in zip(guess, ("f_1", "h1_1", "h2_1")))


def test_set_zk_lookup_argument_checks():
    import plonkathon_b200 as pb
    from plonkathon_b200 import parallel
    p = pb.Prover.__new__(pb.Prover)
    with pytest.raises(ValueError, match="21 blinders"):
        p.set_zk_lookup(True, [1] * 11)
    with pytest.raises(ValueError, match=r"\[0, r\)"):
        p.set_zk_lookup(True, [1] * 20 + [R])
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.__new__(parallel.ShardedProver).set_zk_lookup(True)


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _gpu_prover(pb, c, setup=None, blinders=None, zk=True):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n + 6)
    kw = {"lookups": syn.lookups_arrays(c)} if c.lookups else {"lookup": syn.lookup_arrays(c)}
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c), **kw)
    if zk:
        prover.set_zk_lookup(True, blinders)
    return setup, pk, prover, (A, B, C, public)


def _vk(setup, c, pk):
    kw = {"lookups": syn.lookups_arrays(c)} if c.lookups else {"lookup": syn.lookup_arrays(c)}
    return setup.verification_key_arrays(c.group_order, pk, custom=syn.custom_arrays(c), **kw)


GPU_CASES = [(log_n, p, k) for log_n in (4, 8, 12) for p in (2, 9) for k in (1, 2, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("custom", [(), TERM], ids=["plain", "x2"])
@pytest.mark.parametrize("log_n,n_public,count", GPU_CASES)
def test_gpu_zk_lookup_proof_equals_oracle(log_n, n_public, count, custom):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated"""
    import plonkathon_b200 as pb
    seed = 400 + log_n + n_public + count
    c = _circuit(log_n, n_public, count, custom, seed)
    bl = _blinders(seed)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c, blinders=bl)
    raw = prover.prove_arrays(A, B, C, public)
    _, _, proof, _ = _oracle(c, bl)
    assert len(raw) == 1216
    assert raw == XO.proof_bytes(proof)
    assert prover.prove_arrays(A, B, C, public) == raw  # fixed blinders: the same proof again


def _golden_circuit(rec, tagged):
    if tagged:
        return syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                                 lookups=[range_table(256), xor_table(4), and_table(4)])
    k = rec["table_rows"]
    return syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                             lookup=[list(range(k)), [0] * k, [0] * k])


@pytest.mark.gpu
@pytest.mark.parametrize("name,tagged", [("proof_lookup_2p16.json", False), ("proof_tagged_lookup_2p16.json", True)])
def test_gpu_zero_blinders_reproduce_lookup_goldens(name, tagged):
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, name)))
    c = _golden_circuit(rec, tagged)
    setup = pb.Setup.generate(TAU, c.group_order + 6)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c, setup, [0] * 21)
    assert prover.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]


@pytest.mark.gpu
def test_gpu_golden_zk_lookup_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_zk_lookup_2p16.json")))
    c = _golden_circuit(rec, True)
    n = c.group_order
    setup = pb.Setup.generate(TAU, rec["srs_powers"])
    _, pk, prover, (A, B, C, public) = _gpu_prover(pb, c, setup, [int(b) for b in rec["blinders"]])
    raw = prover.prove_arrays(A, B, C, public)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden zero-knowledge lookup proof"
    vk = _vk(setup, c, pk)
    pf = pb.LookupProof.from_bytes(raw)
    pub = [int(x) for x in rec["public"]]
    assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)


def _tamper_word(raw, k):
    """raw with 32-byte word k (counted from the start of the proof) incremented"""
    x = (int.from_bytes(raw[32 * k:32 * k + 32], "big") + 1) % R
    return raw[:32 * k] + x.to_bytes(32, "big") + raw[32 * k + 32:]


@pytest.mark.gpu
def test_gpu_fresh_blinders_differ_and_verify():
    import plonkathon_b200 as pb
    c = _circuit(10, 2, 3, TERM, 12)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c)
    p1 = prover.prove_arrays(A, B, C, public)
    p2 = prover.prove_arrays(A, B, C, public)
    f1, f2 = XO.proof_from_bytes(p1), XO.proof_from_bytes(p2)
    assert all(f1[k] != f2[k] for k in POINTS)
    vk = _vk(setup, c, pk)
    for raw in (p1, p2):
        pf = pb.LookupProof.from_bytes(raw)
        assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
        bad = pb.LookupProof.from_bytes(_tamper_word(raw, 24 + 8 + 4))  # h1_shifted_eval
        assert not vk.verify_proof(n, bad, public) and not vk.verify_proof_unoptimized(n, bad, public)


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 3])
def test_gpu_round_by_round_equals_whole_proof(count):
    """fixed blinders: the rounds through the C ABI, fed the challenges of the whole proof's transcript, give its bytes"""
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    c = _circuit(8, 2, count, TERM, 21)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c, blinders=_blinders(21))
    raw = prover.prove_arrays(A, B, C, public)
    ch = XO.challenges(XO.proof_from_bytes(raw))
    le = lambda k: (ch[k] % R).to_bytes(32, "little")  # noqa: E731
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    pub = np.ascontiguousarray(np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in public), np.uint8))
    L, h, out = _lib.lib(), prover._h, ctypes.create_string_buffer(1216)
    _lib.check(L.pb200_prover_round1(h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out))
    _lib.check(L.pb200_prover_round_lookup(h, le("eta"), out))
    _lib.check(L.pb200_prover_round2_lookup(h, le("beta"), le("gamma"), le("delta"), le("epsilon"), out))
    _lib.check(L.pb200_prover_round3(h, le("alpha"), le("fft_cofactor"), out))
    _lib.check(L.pb200_prover_round4_lookup(h, le("zeta"), out))
    _lib.check(L.pb200_prover_round5(h, le("v"), out))
    _lib.check(L.pb200_prover_serialize_lookup(h, out))
    assert out.raw == raw


@pytest.mark.gpu
def test_gpu_switching_and_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, parallel
    from plonkathon_b200.lookup import check_lookup
    rec = json.load(open(os.path.join(GOLDEN, "proof_lookup_2p16.json")))
    c = _golden_circuit(rec, False)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c, pb.Setup.generate(TAU, n + 6), zk=False)
    vk = _vk(setup, c, pk)
    golden = lambda: prover.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]  # noqa: E731
    assert golden()
    for off in (lambda: prover.set_zk_lookup(False), lambda: prover.set_zk(False)):
        prover.set_zk_lookup(True)
        raw = prover.prove_arrays(A, B, C, public)
        assert raw.hex() != rec["proof_hex"]
        assert vk.verify_proof(n, pb.LookupProof.from_bytes(raw), public)
        with pytest.raises(RuntimeError, match="T1"):
            prover.T1
        off()
        assert not prover.zk and golden()
    # refusals, each leaving the prover as it was
    L = _lib.lib()
    assert L.pb200_prover_set_zk_lookup(prover._h, 1, b"\xff" * 32 * 21) != 0
    assert "not reduced" in L.pb200_last_error().decode()
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge mode does not combine with lookups"):
        prover.set_zk(True)
    assert golden()
    prover.set_zk_lookup(True, [0] * 21)
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge mode does not combine with lookups"):
        prover.set_zk(True, [0] * 11)
    assert golden()  # still in zero-knowledge lookup mode, with zero blinders
    prover.set_zk_lookup(False)
    plain = pb.Prover.from_arrays(setup, n, pk)
    with pytest.raises(_lib.PlonkB200Error, match="no lookup table"):
        plain.set_zk_lookup(True)
    plain.set_zk(True)
    qk, cols, rows = check_lookup(syn.lookup_arrays(c), n)
    with pytest.raises(_lib.PlonkB200Error, match="lookups do not combine with zero-knowledge"):
        plain._set_lookup(qk, cols, rows)
    assert len(plain.prove_arrays(A, B, C, public)) == 768
    short = pb.Prover.from_arrays(pb.Setup.generate(TAU, n), n, pk, lookup=syn.lookup_arrays(c))
    with pytest.raises(_lib.PlonkB200Error, match=r"n \+ 6"):
        short.set_zk_lookup(True)
    assert short.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]
    tiny = {k: np.zeros((4, 32), np.uint8) for k in pk}
    small = pb.Prover.from_arrays(pb.Setup.generate(TAU, 64), 4, tiny, lookup=([0] * 4, ([0], [0], [0])))
    with pytest.raises(_lib.PlonkB200Error, match="n >= 8"):
        small.set_zk_lookup(True)
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.__new__(parallel.ShardedProver).set_zk_lookup(True)
    assert golden()


@pytest.mark.gpu
def test_gpu_zk_lookup_2p20_verifies():
    """the bench family at 2^20 with a quarter of its rows on three tables"""
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, lookups=[range_table(1 << 16), xor_table(4), and_table(4)])
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c)
    raw = prover.prove_arrays(A, B, C, public)
    vk = _vk(setup, c, pk)
    pf = pb.LookupProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    bad = pb.LookupProof.from_bytes(_tamper_word(raw, 24 + 8))  # f_eval
    assert not vk.verify_proof(n, bad, public) and not vk.verify_proof_unoptimized(n, bad, public)
