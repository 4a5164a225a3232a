"""Shuffles: the rows with q_in = 1 hold the same multiset of (a, b, c) as the rows with q_out = 1
(plonkathon_b200/shuffle.py).

CPU: the oracle with a shuffle (tests/extended_oracle.py) proves circuits at n = 16, 64 and 256, plain and with same-row
or next-row terms, that its trapdoor verifier and both host verifier routines accept; both routines reject tampered
proofs, swapped openings, wrong keys and proofs of the wrong kind; a_1 b_1 c_1 z_1 equal the pinned plain oracle's and
with no shuffled rows z3_1 is the generator; out-rows that are not a permutation raise; the selector checks and the
canonical decoding.  GPU: the prover's 896 and 992 bytes equal the oracle's at several sizes, on both public-input paths
and for a skewed shuffle; the round-by-round ABI gives the same bytes; the 2^16 golden proof is reproduced; a 2^20 proof
verifies; the library refuses what it must and stays usable."""
import ctypes
import json
import os

import numpy as np
import pytest

from oracle import fast as F
from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from tests import extended_oracle as XO
from tests.oracle_keys import host_lincomb  # noqa: F401  (a fixture)
from tests.golden_io import GOLDEN

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
NEXT_TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
TERM_SETS = [[], [(2, 0, 0), (1, 1, 1)], NEXT_TERMS]
TERM_IDS = ["plain", "same_row", "next_row"]
PK_KEYS = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")


def _circuit(log_n, n_public, terms, seed):
    """a synthetic circuit with a shuffle, with at least one shuffled row"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=terms, shuffle=True)
        if any(c.shuffle[0]):
            return c
        seed += 1000


def _oracle_proof(c, fast=True):
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n)
    if not fast:
        setup = O.Setup([setup.point(i) for i in range(n)], None)
    return pk, XO.prove(setup, pk, A, B, C, c.public_values(), fast=fast)


def _oracle_vk(c, pk):
    setup = F.Setup(TAU, c.group_order)
    with F.c_kernels():
        vk = {k: setup.commit(col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                  ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
        custom = [(e, setup.commit(col)) for e, col in c.custom]
        shuffle = tuple(setup.commit(q) if any(q) else None for q in c.shuffle)
    return vk, custom, shuffle


def _host_key(pb, n, vk, custom, shuffle):
    fq = lambda p: None if p is None else (pb.FQ(p[0]), pb.FQ(p[1]))  # noqa: E731
    base = [fq(vk[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")]
    return pb.VerificationKey(n, *base, pb.g2_mul(pb.G2, TAU), pb.Scalar.root_of_unity(n),
                              tuple((e, fq(p)) for e, p in custom), (), tuple(fq(p) for p in shuffle))


def _host_proof(pb, raw):
    return (pb.NextRowShuffleProof if len(raw) == 992 else pb.ShuffleProof).from_bytes(raw)


# ---- CPU: selectors and the circuit builder --------------------------------------------------------------------------
@pytest.mark.parametrize("shuffle,match", [
    (([0] * 15, [0] * 16), "q_in has 15 rows"), (([0] * 16, [0] * 17), "q_out has 17 rows"),
    (([2] + [0] * 15, [0] * 16), "q_in must be 0 or 1"), (([0] * 16, [R - 1] + [0] * 15), "q_out must be 0 or 1"),
    (([1, 1] + [0] * 14, [1] + [0] * 15), "as many q_in rows as q_out rows: 2 and 1"), ((1, 2, 3), "shuffle must be"),
])
def test_malformed_selectors_are_rejected(shuffle, match):
    import plonkathon_b200 as pb
    n = 16
    pk = {k: np.zeros((n, 32), np.uint8) for k in PK_KEYS}
    with pytest.raises(ValueError, match=match):
        pb.Prover.from_arrays(None, n, pk, shuffle=shuffle)
    with pytest.raises(ValueError, match=match):
        pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, shuffle=shuffle)


def test_shuffle_refused_with_lookups_and_on_the_sharded_prover():
    import plonkathon_b200 as pb
    from plonkathon_b200 import parallel
    n = 16
    pk = {k: np.zeros((n, 32), np.uint8) for k in PK_KEYS}
    sh = ([0] * n, [0] * n)
    table = ([1], [2], [3])
    for kw in ({"lookup": ([0] * n, table)}, {"lookups": [([0] * n, table)]}):
        with pytest.raises(ValueError, match="shuffles do not combine with lookups"):
            pb.Prover.from_arrays(None, n, pk, shuffle=sh, **kw)
        with pytest.raises(ValueError, match="shuffles do not combine with lookups"):
            pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, shuffle=sh, **kw)
    with pytest.raises(ValueError, match="shuffles do not combine with lookups"):
        syn.build_circuit(4, lookup=table, shuffle=True)
    with pytest.raises(ValueError, match="sharded"):
        parallel.ShardedProver.from_arrays(None, n, pk, shuffle=sh)


def test_builder_without_shuffle_is_unchanged_and_with_it_shuffles_a_quarter():
    from plonkathon_b200.shuffle import multisets_match
    for terms in TERM_SETS:
        a = syn.build_circuit(8, seed=77, n_public=2, custom=terms)
        b = syn.build_circuit(8, seed=77, n_public=2, custom=terms, shuffle=False)
        assert a.values == b.values and a.QC == b.QC and np.array_equal(a.wire_L, b.wire_L) and b.shuffle == ()
    c = syn.build_circuit(12, seed=5, n_public=2, custom=NEXT_TERMS, shuffle=True)
    q_in, q_out = c.shuffle
    n = c.group_order
    assert sum(q_in) == sum(q_out) and 0.2 * n < sum(q_out) < 0.3 * n
    assert not any(i and o for i, o in zip(q_in, q_out))
    A, B, C = c.wires_values()
    assert multisets_match(A, B, C, q_in, q_out)
    # the out-rows hold the in-rows' tuples in another order
    ins = [(A[i], B[i], C[i]) for i in range(n) if q_in[i]]
    outs = [(A[i], B[i], C[i]) for i in range(n) if q_out[i]]
    assert ins != outs


# ---- CPU: the oracle -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_shuffle_proof_verifies(terms, log_n, host_lincomb):
    pb = host_lincomb
    c = _circuit(log_n, 2, terms, 100 + log_n)
    n = c.group_order
    pk, proof = _oracle_proof(c, fast=log_n > 4)  # 2^4: the pure-Python transforms
    vk, custom, shuffle = _oracle_vk(c, pk)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=custom, shuffle=shuffle), proof, public, TAU)
    assert not XO.verify_proof_trapdoor(n, dict(vk, custom=custom, shuffle=shuffle), proof, [public[0] + 1] + public[1:], TAU)
    key = _host_key(pb, n, vk, custom, shuffle)
    raw = XO.proof_bytes(proof)
    assert len(raw) == (992 if terms == NEXT_TERMS else 896)
    pf = _host_proof(pb, raw)
    assert pf.to_bytes() == raw
    assert key.verify_proof(n, pf, public) and key.verify_proof_unoptimized(n, pf, public)


@pytest.mark.parametrize("terms", TERM_SETS, ids=TERM_IDS)
def test_both_routines_reject_tampered_proofs_and_wrong_keys(terms, host_lincomb):
    pb = host_lincomb
    c = _circuit(4, 2, terms, 21)
    n = c.group_order
    pk, proof = _oracle_proof(c)
    vk, custom, shuffle = _oracle_vk(c, pk)
    good = _host_key(pb, n, vk, custom, shuffle)
    public = c.public_values()
    raw = XO.proof_bytes(proof)
    pf = _host_proof(pb, raw)
    assert good.verify_proof(n, pf, public) and good.verify_proof_unoptimized(n, pf, public)
    bad = {}
    for k in ("qin_eval", "z3_shifted_eval"):
        bad["tampered " + k] = _host_proof(pb, XO.proof_bytes(dict(proof, **{k: (proof[k] + 1) % R})))
    bad["swapped openings"] = _host_proof(pb, XO.proof_bytes(dict(proof, W_z_1=proof["W_zw_1"], W_zw_1=proof["W_z_1"])))
    bad["z3_1 replaced by z_1"] = _host_proof(pb, XO.proof_bytes(dict(proof, z3_1=proof["z_1"])))
    bad["a plain proof"] = pb.Proof.from_bytes(raw[:768])
    if terms == NEXT_TERMS:
        bad["a next-row proof"] = pb.NextRowProof.from_bytes(raw[:864])
    for why, p in bad.items():
        assert not good.verify_proof(n, p, public), why
        assert not good.verify_proof_unoptimized(n, p, public), why
    # a key with [q_in] and [q_out] swapped, and keys without the shuffle
    for why, key in (("swapped selectors", _host_key(pb, n, vk, custom, shuffle[::-1])),
                     ("no shuffle", _host_key(pb, n, vk, custom, ()))):
        assert not key.verify_proof(n, pf, public), why
        assert not key.verify_proof_unoptimized(n, pf, public), why


def test_proof_of_the_other_kind_is_refused(host_lincomb):
    """a shuffle key without next-row terms refuses a NextRowShuffleProof and the reverse"""
    pb = host_lincomb
    c_plain, c_next = _circuit(4, 2, [], 31), _circuit(4, 2, NEXT_TERMS, 31)
    keys, proofs = [], []
    for c in (c_plain, c_next):
        pk, proof = _oracle_proof(c)
        keys.append((_host_key(pb, c.group_order, *_oracle_vk(c, pk)), c.public_values()))
        proofs.append(_host_proof(pb, XO.proof_bytes(proof)))
    for (key, public), pf in ((keys[0], proofs[1]), (keys[1], proofs[0])):
        assert not key.verify_proof(16, pf, public) and not key.verify_proof_unoptimized(16, pf, public)


def test_cross_pins_with_the_pinned_oracle():
    """rounds 1 and 2 are the pinned oracle's (oracle/plonk_oracle.py), and beta, gamma are drawn before theta, kappa:
    a_1 b_1 c_1 z_1 agree.  With no shuffled rows Z3 is the constant 1, so z3_1 is the generator."""
    c = _circuit(6, 2, [(2, 0, 0), (1, 1, 1)], 7)
    n = c.group_order
    pk, proof = _oracle_proof(c)
    plain = O.Prover(F.Setup(TAU, n), pk, check=False)  # its gate check does not know the custom terms
    plain.PI = [(-v) % R for v in c.public_values()] + [0] * (n - len(c.public_values()))
    tr = O.Transcript(b"plonk")
    with F.c_kernels():
        a_1, b_1, c_1 = plain.round_1(*c.wires_values())
        plain.beta, plain.gamma = tr.round_1(a_1, b_1, c_1)
        z_1 = plain.round_2()
    for k, x in (("a_1", a_1), ("b_1", b_1), ("c_1", c_1), ("z_1", z_1)):
        assert proof[k] == x, k
    empty = syn.ArrayCircuit(**{**c.__dict__, "shuffle": ([0] * n, [0] * n)})
    _, proof0 = _oracle_proof(empty)
    assert proof0["z3_1"] == O.G1 and proof0["z3_shifted_eval"] == 1 and proof0["qin_eval"] == 0


def test_out_rows_that_are_not_a_permutation_raise():
    c = _circuit(5, 2, [], 9)
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    r = pk.q_out.index(1)
    A[r] = (A[r] + 1) % R  # an out-row whose a is not the a of its in-row (the row's selectors are all zero)
    with pytest.raises(AssertionError, match="not permutations of each other"):
        XO.prove(F.Setup(TAU, n), pk, A, B, C, c.public_values(), fast=True)


def test_non_canonical_encodings_are_rejected():
    import plonkathon_b200 as pb
    for terms, cls, scalars, points in (([], pb.ShuffleProof, (26, 27), (24, 25)),
                                        (NEXT_TERMS, pb.NextRowShuffleProof, (24, 25, 26, 29, 30), (27, 28))):
        _, proof = _oracle_proof(_circuit(4, 2, terms, 21))
        raw = XO.proof_bytes(proof)
        assert cls.from_bytes(raw).to_bytes() == raw
        for word in scalars + points:
            x = int.from_bytes(raw[32 * word:32 * word + 32], "big") + (R if word in scalars else O.Q_MOD)
            if x >= 1 << 256:
                continue
            with pytest.raises(ValueError, match="word %d" % word):
                cls.from_bytes(raw[:32 * word] + x.to_bytes(32, "big") + raw[32 * word + 32:])
        with pytest.raises(ValueError, match=str(len(raw))):
            cls.from_bytes(raw[:-32])


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _gpu_prover(pb, c, setup=None):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))
    return setup, pk, prover, (A, B, C, public)


GPU_SIZES = [(4, 2), (8, 2), (12, 2), (8, 11), (12, 9)]
GPU_TERMS = TERM_SETS + [list(syn.RUNNING_SUM_TERMS)]
GPU_TERM_IDS = TERM_IDS + ["running_sum"]


@pytest.mark.gpu
@pytest.mark.parametrize("terms", GPU_TERMS, ids=GPU_TERM_IDS)
@pytest.mark.parametrize("log_n,n_public", GPU_SIZES)
def test_gpu_shuffle_proof_equals_oracle(terms, log_n, n_public):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated"""
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, terms, 200 + log_n + n_public)
    _, _, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    _, proof = _oracle_proof(c)
    assert len(raw) == (896 if terms in ([], [(2, 0, 0), (1, 1, 1)]) else 992)
    assert raw == XO.proof_bytes(proof)


def _skewed_circuit(log_n):
    """every in-row holds the same tuple (x, y, x y): in the first half of the rows the even rows are in-rows, copies of
    three variables, and the odd rows out-rows, three fresh variables each; the second half holds fresh random products.
    Every row has the gate c = a b."""
    import random
    n = 1 << log_n
    rng = random.Random(log_n)
    x, y = 12345, R - 678910
    ids = 3 + np.arange(3 * n, dtype=np.int64).reshape(n, 3)
    ids[0:n // 2:2] = (0, 1, 2)
    values = [x, y, x * y % R] * (n // 2 + 1)
    for _ in range(n // 2):
        a, b = rng.randrange(R), rng.randrange(R)
        values += [a, b, a * b % R]
    half = [1, 0] * (n // 4) + [0] * (n // 2)
    return syn.ArrayCircuit(group_order=n, n_constraints=n, wire_L=ids[:, 0].copy(), wire_R=ids[:, 1].copy(),
                            wire_O=ids[:, 2].copy(), QL=[0] * n, QR=[0] * n, QM=[R - 1] * n, QO=[1] * n, QC=[0] * n,
                            n_public=0, values=values, text=[], shuffle=(half, [0] + half[:-1]))


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [4, 8, 12])
def test_gpu_skewed_shuffle_equals_oracle(log_n):
    import plonkathon_b200 as pb
    c = _skewed_circuit(log_n)
    _, _, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    _, proof = _oracle_proof(c)
    assert len(raw) == 896 and raw == XO.proof_bytes(proof)


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [[], NEXT_TERMS], ids=["plain", "next_row"])
def test_gpu_round_by_round_abi_gives_the_whole_proof(terms):
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    from plonkathon_b200.transcript import SHUFFLE_SCHEDULE, Transcript
    c = _circuit(8, 2, terms, 55)
    _, _, prover, (A, B, C, public) = _gpu_prover(pb, c)
    whole = prover.prove_arrays(A, B, C, public)
    tr = Transcript(b"plonk")
    msg_1 = prover.round_1_arrays(A, B, C, public)
    prover.beta, prover.gamma, prover.theta, prover.kappa = tr.round_1(msg_1, SHUFFLE_SCHEDULE)
    msg_2 = prover.round_2()
    prover.alpha, prover.fft_cofactor = tr.round_2(msg_2)
    msg_3 = prover.round_3()
    prover.zeta = tr.round_3(msg_3)
    msg_4 = prover.round_4()
    prover.v = tr.round_4(msg_4)
    msg_5 = prover.round_5()
    m4 = pb.prover.Message4(*[getattr(msg_4, k) for k in pb.prover.PROOF_FIELDS[7:13]])
    plain = pb.Proof(msg_1, pb.prover.Message2(msg_2.z_1), msg_3, m4, msg_5)
    tail = [msg_2.z3_1, msg_4.qin_eval, msg_4.z3_shifted_eval]
    if terms:
        pf = pb.NextRowShuffleProof(plain, msg_4.a_shifted_eval, msg_4.b_shifted_eval, msg_4.c_shifted_eval, *tail)
    else:
        pf = pb.ShuffleProof(plain, *tail)
    assert pf.to_bytes() == whole
    out = ctypes.create_string_buffer(len(whole))
    fn = _lib.lib().pb200_prover_serialize_next_row_shuffle if terms else _lib.lib().pb200_prover_serialize_shuffle
    _lib.check(fn(prover._h, out))
    assert out.raw == whole


@pytest.mark.gpu
def test_gpu_golden_shuffle_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_shuffle_2p16.json")))
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                          custom=[tuple(e) for e in rec["terms"]], shuffle=True)
    assert sum(c.shuffle[0]) == rec["rows_in"]
    n = c.group_order
    setup, pk, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden shuffle proof"
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))
    assert [[str(p[0].n), str(p[1].n)] for p in vk.shuffle] == rec["vk_shuffle"]
    public = [int(x) for x in rec["public"]]
    pf = pb.NextRowShuffleProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_shuffle_2p20_verifies():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, custom=NEXT_TERMS, shuffle=True)
    n = c.group_order
    setup, pk, prover, wires = _gpu_prover(pb, c)
    raw = prover.prove_arrays(*wires)
    vk = setup.verification_key_arrays(n, pk, custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))
    public = c.public_values()
    pf = pb.NextRowShuffleProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    k = 992 - 32  # z3_shifted_eval
    bad = raw[:k] + ((int.from_bytes(raw[k:], "big") + 1) % R).to_bytes(32, "big")
    assert not vk.verify_proof(n, pb.NextRowShuffleProof.from_bytes(bad), public)
    assert not vk.verify_proof_unoptimized(n, pb.NextRowShuffleProof.from_bytes(bad), public)


@pytest.mark.gpu
def test_gpu_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    L = _lib.lib()
    c = _circuit(8, 2, [], 71)
    n = c.group_order
    setup, pk, prover, (A, B, C, public) = _gpu_prover(pb, c)
    good = prover.prove_arrays(A, B, C, public)
    err = lambda: L.pb200_last_error().decode()  # noqa: E731
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    pub = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in public), np.uint8).reshape(-1, 32).copy()
    out = ctypes.create_string_buffer(1216)
    # the entry points of other proof sizes
    assert L.pb200_prover_prove(prover._h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out) != 0
    assert "896 bytes" in err() and "pb200_prover_prove_shuffle" in err()
    assert L.pb200_prover_serialize(prover._h, out) != 0 and "896 bytes" in err()
    assert L.pb200_prover_round2(prover._h, bytes(32), bytes(32), out) != 0 and "round2_shuffle" in err()
    assert L.pb200_prover_round4(prover._h, bytes(32), out) != 0 and "round4_shuffle" in err()
    assert L.pb200_prover_prove_next_row_shuffle(prover._h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out) != 0
    assert "pb200_prover_prove_shuffle" in err()
    assert L.pb200_prover_serialize_next_row_shuffle(prover._h, out) != 0
    assert L.pb200_prover_round4_next_row_shuffle(prover._h, bytes(32), out) != 0
    # the plain and next-row entry points on a next-row shuffle prover, and the shuffle ones on a plain prover
    cn = _circuit(8, 2, NEXT_TERMS, 72)
    _, _, nprover, (An, Bn, Cn, pn) = _gpu_prover(pb, cn, setup)
    pubn = np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in pn), np.uint8).reshape(-1, 32).copy()
    assert L.pb200_prover_prove_next_row(nprover._h, ptr(An), ptr(Bn), ptr(Cn), ptr(pubn), len(pn), out) != 0
    assert "992 with next-row terms" in err() and "pb200_prover_prove_next_row_shuffle" in err()
    assert L.pb200_prover_prove_shuffle(nprover._h, ptr(An), ptr(Bn), ptr(Cn), ptr(pubn), len(pn), out) != 0
    assert "next-row" in err()
    plain = pb.Prover.from_arrays(setup, n, pk)
    assert L.pb200_prover_prove_shuffle(plain._h, ptr(A), ptr(B), ptr(C), ptr(pub), len(public), out) != 0
    assert "no shuffle" in err()
    # lookups and zero knowledge on a shuffle prover, a shuffle on a zero-knowledge or lookup prover
    with pytest.raises(_lib.PlonkB200Error, match="do not combine with a shuffle"):
        prover._set_lookup([0] * n, ([1], [2], [3]), 1)
    with pytest.raises(_lib.PlonkB200Error, match="does not combine with a shuffle"):
        prover.set_zk(True)
    zk = pb.Prover.from_arrays(pb.Setup.generate(TAU, n + 6), n, pk)
    zk.set_zk(True)
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge"):
        zk._set_shuffle(*syn.shuffle_arrays(c))
    lk = pb.Prover.from_arrays(setup, n, pk)
    lk._set_lookup([0] * n, ([1], [2], [3]), 1)
    with pytest.raises(_lib.PlonkB200Error, match="lookups"):
        lk._set_shuffle(*syn.shuffle_arrays(c))
    # selectors set twice, and selectors the library checks itself (the Python checks come first otherwise)
    with pytest.raises(_lib.PlonkB200Error, match="already set"):
        prover._set_shuffle(*syn.shuffle_arrays(c))
    fresh = pb.Prover.from_arrays(setup, n, pk)
    with pytest.raises(_lib.PlonkB200Error, match="q_in must be 0 or 1"):
        fresh._set_shuffle([2] + [0] * (n - 1), [0] * n)
    with pytest.raises(_lib.PlonkB200Error, match="as many q_in rows as q_out rows"):
        fresh._set_shuffle([1] + [0] * (n - 1), [0] * n)
    assert not getattr(fresh, "shuffle", False)
    assert len(fresh.prove_arrays(A, B, C, public)) == 768  # a refused call left it a plain prover
    # a witness whose out-rows are not a permutation of its in-rows
    bad = A.copy()
    r = c.shuffle[1].index(1)
    bad[r] = np.frombuffer(((int.from_bytes(A[r].tobytes(), "little") + 1) % R).to_bytes(32, "little"), np.uint8)
    with pytest.raises(AssertionError, match="shuffle: the q_in rows and the q_out rows are not permutations"):
        prover.prove_arrays(bad, B, C, public)
    # every refused call left the prover usable
    assert prover.prove_arrays(A, B, C, public) == good
