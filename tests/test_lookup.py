"""Lookups: a plookup argument over one fixed three-column table (plonkathon_b200/lookup.py).

CPU: the oracle with a lookup argument (tests/extended_oracle.py) proves circuits that its trapdoor verifier and the
product's host verifier accept, for a padded range table, a 4-bit XOR table that fills the domain and a table with
duplicate rows, each with and without a custom term; the verifiers reject tampered proofs, wrong keys and plain proofs;
malformed arguments are refused.  GPU: the prover's 1216 bytes equal the oracle's, the 2^16 golden lookup proof is
reproduced, a 2^20 lookup circuit verifies, and the combinations that are out of scope are refused."""
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
from tests.golden_io import GOLDEN

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
TERM = [(2, 0, 0)]


def range_table(n):
    """0 .. n/2 - 1 in t1, zero t2 and t3: shorter than n (padded), two constant-zero columns"""
    k = max(2, n // 2)
    return [list(range(k)), [0] * k, [0] * k]


def xor_table():
    """(x, y, x ^ y) for 4-bit x, y: 256 rows"""
    rows = [(x, y, x ^ y) for x in range(16) for y in range(16)]
    return [list(c) for c in zip(*rows)]


def dup_table():
    """rows 0 and 2, 1 and 4 are equal"""
    rows = [(11, 12, 13), (21, 22, 23), (11, 12, 13), (31, 32, 33), (21, 22, 23), (41, 42, 43)]
    return [list(c) for c in zip(*rows)]


TABLES = {"range": range_table, "xor": lambda n: xor_table(), "dup": lambda n: dup_table()}


def _circuit(log_n, n_public, table, custom, seed):
    """the first synthetic circuit from ``seed`` on that has lookup rows (and uses the custom term)"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=custom, lookup=table)
        if any(c.lookup[0]) and all(any(col) for _, col in c.custom):
            return c
        seed += 1000


def _commit_col(setup, col):
    if not any(col):
        return None  # a constant-zero column commits to the identity
    with F.c_kernels():
        return setup.commit(col)


def _oracle(c, fast=True):
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, n)
    proof = XO.prove(setup, pk, A, B, C, c.public_values(), fast=fast)
    return pk, setup, proof


def _oracle_vk(c, pk, setup):
    vk = {k: _commit_col(setup, col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO),
                                                    ("Qc", c.QC), ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom = [(e, _commit_col(setup, col)) for e, col in c.custom]
    lookup = tuple(_commit_col(setup, col) for col in [pk.qk] + pk.table)
    return vk, custom, lookup


def _host_vk(pb, c, vk, custom, lookup):
    fq = lambda p: None if p is None else (pb.FQ(p[0]), pb.FQ(p[1]))  # noqa: E731
    n = c.group_order
    base = [fq(vk[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")]
    return pb.VerificationKey(n, *base, pb.g2_mul(pb.G2, TAU), pb.Scalar.root_of_unity(n),
                              tuple((e, fq(p)) for e, p in custom), tuple(fq(p) for p in lookup))


# ---- CPU ---------------------------------------------------------------------------------------------------------
CPU_CASES = [(log_n, t) for log_n in (4, 6, 8) for t in ("range", "dup")] + [(8, "xor")]


@pytest.mark.parametrize("custom", [(), TERM], ids=["plain", "x2"])
@pytest.mark.parametrize("log_n,table", CPU_CASES)
def test_oracle_lookup_proof_verifies(log_n, table, custom, host_lincomb):
    pb = host_lincomb
    n = 1 << log_n
    c = _circuit(log_n, 2, TABLES[table](n), custom, 300 + log_n)
    pk, setup, proof = _oracle(c, fast=log_n > 4)  # 2^4: the pure-Python transforms
    vk, cpts, lpts = _oracle_vk(c, pk, setup)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), proof, public, TAU)
    key = _host_vk(pb, c, vk, cpts, lpts)
    pf = pb.LookupProof.from_bytes(XO.proof_bytes(proof))
    assert key.verify_proof(n, pf, public) and key.verify_proof_unoptimized(n, pf, public)
    if log_n == 4:
        # rejected: tampered evaluations, a wrong public input, a key whose table differs in one entry, a plain proof
        for f in ("f_eval", "h2_eval", "z2_shifted_eval"):
            bad = dict(proof, **{f: (proof[f] + 1) % R})
            assert not XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), bad, public, TAU), f
            bpf = pb.LookupProof.from_bytes(XO.proof_bytes(bad))
            assert not key.verify_proof(n, bpf, public) and not key.verify_proof_unoptimized(n, bpf, public), f
        wrong_pub = [public[0] + 1] + public[1:]
        assert not XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), proof, wrong_pub, TAU)
        assert not key.verify_proof(n, pf, wrong_pub) and not key.verify_proof_unoptimized(n, pf, wrong_pub)
        t1 = list(pk.table[0])
        t1[1] = (t1[1] + 1) % R
        bad_t1 = _commit_col(setup, t1)
        other = dataclasses.replace(key, lookup=(key.lookup[0], (pb.FQ(bad_t1[0]), pb.FQ(bad_t1[1])), *key.lookup[2:]))
        assert not other.verify_proof(n, pf, public) and not other.verify_proof_unoptimized(n, pf, public)
        assert not XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=(lpts[0], bad_t1) + lpts[2:]), proof, public,
                                            TAU)


def test_plain_proof_against_lookup_key_and_reverse(host_lincomb):
    pb = host_lincomb
    c = _circuit(4, 2, range_table(16), (), 41)
    n = c.group_order
    pk, setup, proof = _oracle(c, fast=False)
    vk, cpts, lpts = _oracle_vk(c, pk, setup)
    key = _host_vk(pb, c, vk, cpts, lpts)
    plain_key = dataclasses.replace(key, lookup=())
    lpf = pb.LookupProof.from_bytes(XO.proof_bytes(proof))
    ppf = lpf.plain  # the plain part of a lookup proof: a 768-byte proof of the wrong kind
    public = c.public_values()
    assert not key.verify_proof(n, ppf, public) and not key.verify_proof_unoptimized(n, ppf, public)
    assert not plain_key.verify_proof(n, lpf, public) and not plain_key.verify_proof_unoptimized(n, lpf, public)


def test_oracle_row_outside_the_table_raises():
    c = _circuit(5, 2, dup_table(), (), 5)
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    row = next(i for i in range(c.group_order) if c.lookup[0][i])
    C[row] = (C[row] + 1) % R
    with pytest.raises(AssertionError, match="lookup row %d is not in the table" % row):
        XO.prove(F.Setup(TAU, c.group_order), pk, A, B, C, c.public_values(), fast=True)


def test_oracle_grand_product_closes():
    c = _circuit(5, 2, range_table(32), (), 6)
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    prover = XO.Prover(F.Setup(TAU, c.group_order), pk)
    with F.c_kernels():
        prover.prove(A, B, C, c.public_values())
    # Z2 starts at 1 and its last step returns to 1 (Z2_n = Z2_0)
    n, d, e = c.group_order, prover.delta, prover.epsilon
    od, eod = (1 + d) % R, e * (1 + d) % R
    i = n - 1
    num = od * (e + prover.F[i]) % R * (eod + prover.Tl[i] + d * prover.Tl[0]) % R
    den = (eod + prover.H1[i] + d * prover.H2[i]) * (eod + prover.H2[i] + d * prover.H1[0]) % R
    assert prover.Z2[0] == 1 and prover.Z2[i] * num % R * pow(den, -1, R) % R == 1


def _pk16():
    n = 16
    return n, {k: np.zeros((n, 32), np.uint8) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")}


@pytest.mark.parametrize("lookup,match", [
    (([2] + [0] * 15, ([1], [2], [3])), "0 or 1"),
    (([0] * 16, ([], [], [])), "empty"),
    (([0] * 16, (list(range(17)), [0] * 17, [0] * 17)), "more than"),
    (([0] * 16, ([1, 2], [1], [1, 2])), "unequal"),
    (([0] * 16, ([R], [0], [0])), r"\[0, r\)"),
    (([0] * 16, ([1], [2])), "three columns"),
])
def test_malformed_lookup_is_rejected(lookup, match):
    import plonkathon_b200 as pb
    n, pk = _pk16()
    with pytest.raises(ValueError, match=match):
        pb.Prover.from_arrays(None, n, pk, lookup=lookup)
    with pytest.raises(ValueError, match=match):
        pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, lookup=lookup)


def test_lookup_proof_bytes_round_trip():
    import plonkathon_b200 as pb
    c = _circuit(4, 2, dup_table(), (), 7)
    _, _, proof = _oracle(c, fast=False)
    raw = XO.proof_bytes(proof)
    assert len(raw) == 1216
    pf = pb.LookupProof.from_bytes(raw)
    assert pf.to_bytes() == raw
    assert list(pf.flatten()) == list(XO.proof_fields(("lookup",)))
    for word, bound in ((24, pb.FIELD_MODULUS), (33, R)):  # f_1.x and t_eval
        bad = raw[:32 * word] + bound.to_bytes(32, "big") + raw[32 * word + 32:]
        with pytest.raises(ValueError, match="non-canonical"):
            pb.LookupProof.from_bytes(bad)
    with pytest.raises(ValueError, match="1216"):
        pb.LookupProof.from_bytes(raw[:768])


def test_lookup_keyword_off_keeps_the_plain_circuit():
    a = syn.build_circuit(9, seed=20260924, n_public=2)
    b = syn.build_circuit(9, seed=20260924, n_public=2, lookup=None)
    for f in dataclasses.fields(a):
        x, y = getattr(a, f.name), getattr(b, f.name)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f.name
    assert a.lookup == ()


def test_lookup_rows_have_zero_gate_selectors_and_are_copied_on():
    c = syn.build_circuit(8, seed=3, n_public=2, lookup=range_table(256))
    qk = c.lookup[0]
    rows = [i for i in range(c.group_order) if qk[i]]
    assert rows and len(rows) > c.group_order // 8
    for i in rows:
        assert (c.QL[i], c.QR[i], c.QM[i], c.QO[i], c.QC[i]) == (0, 0, 0, 0, 0)
    looked_up = {int(v) for i in rows for v in (c.wire_L[i], c.wire_R[i], c.wire_O[i])}
    later = {int(v) for i in range(c.n_constraints) if not qk[i] for v in (c.wire_L[i], c.wire_R[i])}
    assert looked_up & later


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _gpu_proof(pb, c, lookup=None, setup=None):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c),
                                   lookup=lookup or syn.lookup_arrays(c))
    return setup, pk, prover, prover.prove_arrays(A, B, C, public)


GPU_CASES = [(log_n, p, t) for log_n in (4, 8, 12) for p in (2, 9) for t in ("range", "xor", "dup")
             if not (t == "xor" and log_n < 8)]


@pytest.mark.gpu
@pytest.mark.parametrize("custom", [(), TERM], ids=["plain", "x2"])
@pytest.mark.parametrize("log_n,n_public,table", GPU_CASES)
def test_gpu_lookup_proof_equals_oracle(log_n, n_public, table, custom):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated"""
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, TABLES[table](1 << log_n), custom, 500 + log_n + n_public)
    _, _, _, raw = _gpu_proof(pb, c)
    _, _, proof = _oracle(c)
    assert len(raw) == 1216
    assert raw == XO.proof_bytes(proof)


@pytest.mark.gpu
def test_gpu_skewed_lookup_equals_oracle():
    """every non-lookup row uses entry 0, every lookup row entry 1: one hot counter each"""
    import plonkathon_b200 as pb
    c = syn.build_circuit(12, seed=77, n_public=2, lookup=([5], [6], [7]))
    table = ([1, 5], [2, 6], [3, 7])
    c = dataclasses.replace(c, lookup=(c.lookup[0], table))
    _, _, _, raw = _gpu_proof(pb, c)
    _, _, proof = _oracle(c)
    assert raw == XO.proof_bytes(proof)


@pytest.mark.gpu
def test_gpu_golden_lookup_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_lookup_2p16.json")))
    k = rec["table_rows"]
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                          lookup=[list(range(k)), [0] * k, [0] * k])
    n = c.group_order
    setup, pk, _, raw = _gpu_proof(pb, c)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden lookup proof"
    vk = setup.verification_key_arrays(n, pk, lookup=syn.lookup_arrays(c))
    assert [None if p is None else [str(p[0].n), str(p[1].n)] for p in vk.lookup] == rec["vk_lookup"]
    pf = pb.LookupProof.from_bytes(raw)
    public = [int(x) for x in rec["public"]]
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_lookup_2p20_verifies_and_rejects():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, lookup=range_table(1 << 16))
    n = c.group_order
    setup, pk, prover, raw = _gpu_proof(pb, c)
    vk = setup.verification_key_arrays(n, pk, lookup=syn.lookup_arrays(c))
    public = c.public_values()
    pf = pb.LookupProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    k = 768 + 4 * 64 + 32 * 5  # z2_shifted_eval, the last word
    bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not vk.verify_proof(n, pb.LookupProof.from_bytes(bad), public)
    assert not vk.verify_proof_unoptimized(n, pb.LookupProof.from_bytes(bad), public)
    _, A, B, C, _ = syn.circuit_arrays(c)
    row = next(i for i in range(n) if c.lookup[0][i])
    A2 = A.copy()
    A2[row] = 0
    A2[row, 0] = 0xFF
    A2[row, 1] = 0xFF  # 65535 + ... : outside the 16-bit range table
    A2[row, 2] = 0x01
    with pytest.raises(AssertionError, match="lookup row %d is not in the table" % row):
        prover.prove_arrays(A2, B, C, public)
    assert prover.prove_arrays(A, B, C, public) == raw  # the prover is still usable


@pytest.mark.gpu
def test_gpu_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, parallel
    c = _circuit(8, 2, range_table(256), (), 11)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n + 8)
    prover = pb.Prover.from_arrays(setup, n, pk, lookup=syn.lookup_arrays(c))
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge mode does not combine with lookups"):
        prover.set_zk(True)
    zk = pb.Prover.from_arrays(setup, n, pk)
    zk.set_zk(True)
    with pytest.raises(_lib.PlonkB200Error, match="lookups do not combine with zero-knowledge"):
        zk._set_lookup([1 if x else 0 for x in c.lookup[0]], [list(t) for t in c.lookup[1]], len(c.lookup[1][0]))
    with pytest.raises(ValueError, match="sharded prover"):
        parallel.ShardedProver.from_arrays(setup, n, pk, lookup=syn.lookup_arrays(c))
    L = _lib.lib()
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    out = ctypes.create_string_buffer(1216)
    for name, call in (
            ("pb200_prover_prove_lookup", lambda: L.pb200_prover_prove(prover._h, ptr(A), ptr(B), ptr(C), None, 0, out)),
            ("pb200_prover_prove_lookup", lambda: L.pb200_prover_prove_device(prover._h, None, None, None, None, 0, out)),
            ("pb200_prover_serialize_lookup", lambda: L.pb200_prover_serialize(prover._h, out)),
            ("pb200_prover_round2_lookup", lambda: L.pb200_prover_round2(prover._h, bytes(32), bytes(32), out)),
            ("pb200_prover_round4_lookup", lambda: L.pb200_prover_round4(prover._h, bytes(32), out))):
        assert call() != 0
        assert name in L.pb200_last_error().decode()
    # a second table, and the plain prover keeps its 768-byte entry points
    assert L.pb200_prover_set_lookup(prover._h, ptr(A), ptr(A), ptr(A), ptr(A), 1) != 0
    assert "already set" in L.pb200_last_error().decode()
    assert len(zk.prove_arrays(A, B, C, public)) == 768
    # and the lookup prover proves round by round through its own entry points
    raw = prover.prove_arrays(A, B, C, public)
    buf = ctypes.create_string_buffer(1216)
    _lib.check(L.pb200_prover_serialize_lookup(prover._h, buf))
    assert buf.raw == raw
