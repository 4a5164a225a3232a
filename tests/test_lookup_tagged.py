"""Lookups over several tables, told apart by a table tag (plonkathon_b200/lookup.py, ``lookups=``).

CPU: the oracle (tests/extended_oracle.py, with Q_T and t4) proves circuits with two and
three tables that its trapdoor verifier and both host verifier routines accept; they reject a tampered evaluation, a
key whose [Q_T] or [t4] carries another assignment of table ids and a key without the two tag commitments.  One table
through ``lookups=`` gives the bytes of the untagged proof with ``lookup=``.  A row tagged XOR whose (a, b, c) is an AND row is refused, while the same witness against the
merged untagged table proves and verifies: the tag is what makes several tables sound.  Malformed arguments are
refused.  GPU: the prover's 1216 bytes equal the oracle's, both golden lookup proofs are reproduced, a 2^20 three-table
circuit verifies, and the refusals of ``pb200_prover_set_lookup_tagged`` hold."""
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
from tests.golden_io import GOLDEN
from tests.oracle_keys import host_lincomb  # noqa: F401  (a fixture)
from tests.test_lookup import _commit_col, _host_vk

R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
TERM = [(2, 0, 0)]


def range_table(k):
    """(v, 0, 0), v < k"""
    return [list(range(k)), [0] * k, [0] * k]


def op_table(bits, op):
    """(x, y, op(x, y)) for x, y < 2^bits"""
    rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(c) for c in zip(*rows)]


def xor_table(bits):
    return op_table(bits, lambda x, y: x ^ y)


def and_table(bits):
    return op_table(bits, lambda x, y: x & y)


def tables(n, count):
    """two tables: XOR and AND; three: a range table first.  Operand widths grow with n and the tables fit in n rows."""
    bits = 1 if n <= 16 else 2 if n <= 64 else 3 if n <= 256 else 4
    out = [range_table(max(2, n // 8)), xor_table(bits), and_table(bits)]
    return out[3 - count:]


def _circuit(log_n, n_public, tabs, custom, seed):
    """the first synthetic circuit from ``seed`` on in which every table has lookup rows (and the custom term is
    used)"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=custom, lookups=tabs)
        if all(any(q) for q, _ in c.lookups) and all(any(col) for _, col in c.custom):
            return c
        seed += 1000


def _oracle(c, fast=True):
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    setup = F.Setup(TAU, c.group_order)
    return pk, setup, XO.prove(setup, pk, A, B, C, c.public_values(), fast=fast)


def _oracle_vk(c, pk, setup):
    vk = {k: _commit_col(setup, col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO),
                                                    ("Qc", c.QC), ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom = [(e, _commit_col(setup, col)) for e, col in c.custom]
    lookup = tuple(_commit_col(setup, col) for col in [pk.qk] + pk.table + [pk.qtag, pk.t4])
    return vk, custom, lookup


def _relabelled(pk, count):
    """Q_T and t4 with table k given id k + 1 mod count: the same tables under another assignment of ids"""
    qt = [(x + 1) % count if q else 0 for q, x in zip(pk.qk, pk.qtag)]
    t4 = [(x + 1) % count for x in pk.t4]
    return qt, t4


# ---- CPU ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("custom", [(), TERM], ids=["plain", "x2"])
@pytest.mark.parametrize("count", [2, 3])
@pytest.mark.parametrize("log_n", [4, 6, 8])
def test_oracle_tagged_proof_verifies(log_n, count, custom, host_lincomb):
    pb = host_lincomb
    n = 1 << log_n
    c = _circuit(log_n, 2, tables(n, count), custom, 700 + log_n + count)
    pk, setup, proof = _oracle(c, fast=log_n > 4)  # 2^4: the pure-Python transforms
    assert any(pk.qtag) and any(pk.t4)
    vk, cpts, lpts = _oracle_vk(c, pk, setup)
    public = c.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), proof, public, TAU)
    key = _host_vk(pb, c, vk, cpts, lpts)
    assert len(key.lookup) == 6
    pf = pb.LookupProof.from_bytes(XO.proof_bytes(proof))
    assert key.verify_proof(n, pf, public) and key.verify_proof_unoptimized(n, pf, public)
    if log_n != 4:
        return
    # rejected: a tampered f_eval, [Q_T] or [t4] of another assignment of ids, a key without the tag commitments
    bad = dict(proof, f_eval=(proof["f_eval"] + 1) % R)
    assert not XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), bad, public, TAU)
    bpf = pb.LookupProof.from_bytes(XO.proof_bytes(bad))
    assert not key.verify_proof(n, bpf, public) and not key.verify_proof_unoptimized(n, bpf, public)
    fq = lambda p: None if p is None else (pb.FQ(p[0]), pb.FQ(p[1]))  # noqa: E731
    qt2, t42 = (_commit_col(setup, col) for col in _relabelled(pk, count))
    for k, pt in ((4, qt2), (5, t42)):
        wrong = lpts[:k] + (pt,) + lpts[k + 1:]
        assert not XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=wrong), proof, public, TAU), k
        other = dataclasses.replace(key, lookup=tuple(fq(p) for p in wrong))
        assert not other.verify_proof(n, pf, public) and not other.verify_proof_unoptimized(n, pf, public), k
    assert not XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts[:4]), proof, public, TAU)
    untagged = dataclasses.replace(key, lookup=key.lookup[:4])
    assert not untagged.verify_proof(n, pf, public) and not untagged.verify_proof_unoptimized(n, pf, public)


@pytest.mark.parametrize("log_n", [4, 8])
def test_one_table_through_lookups_is_the_untagged_proof(log_n):
    n = 1 << log_n
    table = xor_table(2) if log_n == 8 else range_table(8)
    a = syn.build_circuit(log_n, seed=31, n_public=2, lookup=table)
    b = syn.build_circuit(log_n, seed=31, n_public=2, lookups=[table])
    assert a.values == b.values and b.lookups == (a.lookup,)
    assert all(np.array_equal(getattr(a, w), getattr(b, w)) for w in ("wire_L", "wire_R", "wire_O"))
    pk_b = XO.preprocessed(b)
    assert pk_b.qtag == [0] * n and pk_b.t4 == [0] * n
    pa = XO.prove(F.Setup(TAU, n), XO.preprocessed(a), *a.wires_values(), a.public_values(), fast=log_n > 4)
    _, _, pb_ = _oracle(b, fast=log_n > 4)
    assert XO.proof_bytes(pa) == XO.proof_bytes(pb_)  # the untagged oracle's proof


def _swap_row_to(c, row, abc):
    """c with lookup row ``row`` given three fresh variables of values abc: every other constraint still holds"""
    nv = len(c.values)
    wires = [w.copy() for w in (c.wire_L, c.wire_R, c.wire_O)]
    for k in range(3):
        wires[k][row] = nv + k
    return dataclasses.replace(c, values=c.values + list(abc), wire_L=wires[0], wire_R=wires[1], wire_O=wires[2])


def test_tag_keeps_an_xor_row_out_of_the_and_table(host_lincomb):
    pb = host_lincomb
    log_n, n = 6, 64
    xor, and_ = xor_table(2), and_table(2)
    c = _circuit(log_n, 2, [xor, and_], (), 11)
    row = next(i for i in range(n) if c.lookups[0][0][i])  # a row tagged XOR
    abc = (1, 1, 1)  # 1 & 1 = 1, an AND row; 1 ^ 1 = 0, not an XOR row
    assert abc in set(zip(*and_)) and abc not in set(zip(*xor))
    bad = _swap_row_to(c, row, abc)
    with pytest.raises(AssertionError, match="lookup row %d is not in the table" % row):
        _oracle(bad)
    # the same witness against the two tables merged without a tag: it proves and verifies
    merged_q = [x | y for x, y in zip(c.lookups[0][0], c.lookups[1][0])]
    merged = dataclasses.replace(bad, lookups=(), lookup=(merged_q, tuple(x + y for x, y in zip(xor, and_))))
    pk, setup, proof = _oracle(merged)
    vk, cpts, lpts = _oracle_vk(merged, pk, setup)
    lpts = lpts[:4]
    public = merged.public_values()
    assert XO.verify_proof_trapdoor(n, dict(vk, custom=cpts, lookup=lpts), proof, public, TAU)
    key = _host_vk(pb, merged, vk, cpts, lpts)
    pf = pb.LookupProof.from_bytes(XO.proof_bytes(proof))
    assert key.verify_proof(n, pf, public) and key.verify_proof_unoptimized(n, pf, public)


def test_check_lookups_ids_and_layout():
    from plonkathon_b200.lookup import check_lookups
    n = 16
    q0, q1 = [0] * n, [0] * n
    q0[2], q1[5], q1[7] = 1, 1, 1
    qk, qtag, cols, rows = check_lookups([(q0, ([1, 2], [3, 4], [5, 6])), (q1, ([7], [8], [9]))], n)
    assert rows == 3 and cols == [[1, 2, 7], [3, 4, 8], [5, 6, 9], [0, 0, 1]]
    assert [i for i in range(n) if qk[i]] == [2, 5, 7] and (qtag[2], qtag[5], qtag[7]) == (0, 1, 1)
    assert sum(qtag) == 2


def _pk16():
    n = 16
    return n, {k: np.zeros((n, 32), np.uint8) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")}


def _both(n, pk, match, **kw):
    import plonkathon_b200 as pb
    with pytest.raises(ValueError, match=match):
        pb.Prover.from_arrays(None, n, pk, **kw)
    with pytest.raises(ValueError, match=match):
        pb.Setup.__new__(pb.Setup).verification_key_arrays(n, pk, **kw)


def test_malformed_lookups_are_rejected():
    n, pk = _pk16()
    q0, q1 = [0] * n, [0] * n
    q0[3] = q1[3] = 1
    t = ([1], [2], [3])
    _both(n, pk, "overlap on row 3", lookups=[(q0, t), (q1, t)])
    _both(n, pk, "rows in all", lookups=[([0] * n, (list(range(9)), [0] * 9, [0] * 9))] * 2)
    _both(n, pk, "not both", lookup=([0] * n, t), lookups=[([0] * n, t)])
    _both(n, pk, "at least one table", lookups=[])
    _both(n, pk, "0 or 1", lookups=[([0] * n, t), ([2] + [0] * 15, t)])  # each table as lookup= checks it
    _both(n, pk, "three columns", lookups=[([0] * n, ([1], [2]))])
    with pytest.raises(ValueError, match="not both"):
        syn.build_circuit(4, lookup=t, lookups=[t])
    with pytest.raises(ValueError, match="rows in all"):
        syn.build_circuit(4, lookups=[range_table(9), range_table(8)])


def test_lookups_keyword_off_keeps_the_plain_circuit():
    a = syn.build_circuit(9, seed=20260924, n_public=2)
    b = syn.build_circuit(9, seed=20260924, n_public=2, lookups=None)
    for f in dataclasses.fields(a):
        x, y = getattr(a, f.name), getattr(b, f.name)
        assert (np.array_equal(x, y) if isinstance(x, np.ndarray) else x == y), f.name
    assert a.lookups == ()


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _gpu_proof(pb, c, setup=None):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=syn.custom_arrays(c), lookups=syn.lookups_arrays(c))
    return setup, pk, prover, prover.prove_arrays(A, B, C, public)


GPU_CASES = [(log_n, p, k) for log_n in (4, 8, 12) for p in (2, 9) for k in (2, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("custom", [(), TERM], ids=["plain", "x2"])
@pytest.mark.parametrize("log_n,n_public,count", GPU_CASES)
def test_gpu_tagged_lookup_proof_equals_oracle(log_n, n_public, count, custom):
    """<= 8 public inputs: PI from cached Lagrange-basis vectors; > 8: PI interpolated"""
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, tables(1 << log_n, count), custom, 900 + log_n + n_public + count)
    _, _, _, raw = _gpu_proof(pb, c)
    _, _, proof = _oracle(c)
    assert len(raw) == 1216
    assert raw == XO.proof_bytes(proof)


@pytest.mark.gpu
def test_gpu_one_table_through_lookups_reproduces_the_lookup_golden():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_lookup_2p16.json")))
    k = rec["table_rows"]
    table = [list(range(k)), [0] * k, [0] * k]
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"], lookups=[table])
    setup, pk, _, raw = _gpu_proof(pb, c)
    assert raw.hex() == rec["proof_hex"], "one table through lookups= differs from the golden lookup proof"
    n = c.group_order
    vk = setup.verification_key_arrays(n, pk, lookups=syn.lookups_arrays(c))
    assert [None if p is None else [str(p[0].n), str(p[1].n)] for p in vk.lookup] == rec["vk_lookup"] + [None, None]
    pf = pb.LookupProof.from_bytes(raw)
    public = [int(x) for x in rec["public"]]
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_golden_tagged_lookup_proof_2p16():
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_tagged_lookup_2p16.json")))
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                          lookups=[range_table(256), xor_table(4), and_table(4)])
    n = c.group_order
    setup, pk, _, raw = _gpu_proof(pb, c)
    assert raw.hex() == rec["proof_hex"], "GPU proof differs from the oracle's golden tagged lookup proof"
    vk = setup.verification_key_arrays(n, pk, lookups=syn.lookups_arrays(c))
    assert [None if p is None else [str(p[0].n), str(p[1].n)] for p in vk.lookup] == rec["vk_lookup"]
    pf = pb.LookupProof.from_bytes(raw)
    public = [int(x) for x in rec["public"]]
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_tagged_2p20_verifies_and_rejects():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, lookups=[range_table(1 << 16), xor_table(4), and_table(4)])
    n = c.group_order
    setup, pk, prover, raw = _gpu_proof(pb, c)
    vk = setup.verification_key_arrays(n, pk, lookups=syn.lookups_arrays(c))
    public = c.public_values()
    pf = pb.LookupProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    k = 768 + 4 * 64  # f_eval, the first lookup evaluation
    bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not vk.verify_proof(n, pb.LookupProof.from_bytes(bad), public)
    assert not vk.verify_proof_unoptimized(n, pb.LookupProof.from_bytes(bad), public)
    # a row tagged XOR holding (1, 1, 1): a row of the AND table, not of the XOR table
    _, A, B, C, _ = syn.circuit_arrays(c)
    row = next(i for i in range(n) if c.lookups[1][0][i])
    A2, B2, C2 = A.copy(), B.copy(), C.copy()
    for W in (A2, B2, C2):
        W[row] = 0
        W[row, 0] = 1
    with pytest.raises(AssertionError, match="lookup row %d is not in the table" % row):
        prover.prove_arrays(A2, B2, C2, public)
    assert prover.prove_arrays(A, B, C, public) == raw  # the prover is still usable


@pytest.mark.gpu
def test_gpu_tagged_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib, parallel
    from plonkathon_b200.lookup import check_lookups, to_le_rows
    c = _circuit(8, 2, tables(256, 3), (), 13)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n + 8)
    L = _lib.lib()
    qk, qtag, cols, rows = check_lookups(syn.lookups_arrays(c), n)
    off = next(i for i in range(n) if not qk[i])
    bad_tag = list(qtag)
    bad_tag[off] = 1
    keep = [to_le_rows(x) for x in [qk, bad_tag] + cols]
    ptr = [k.ctypes.data_as(ctypes.c_void_p) for k in keep]
    fresh = pb.Prover.from_arrays(setup, n, pk)
    assert L.pb200_prover_set_lookup_tagged(fresh._h, *ptr, rows) != 0
    assert "Q_T must be 0 where q_K = 0: row %d" % off in L.pb200_last_error().decode()
    zk = pb.Prover.from_arrays(setup, n, pk)
    zk.set_zk(True)
    with pytest.raises(_lib.PlonkB200Error, match="lookups do not combine with zero-knowledge"):
        zk._set_lookup_tagged(qk, qtag, cols, rows)
    prover = pb.Prover.from_arrays(setup, n, pk, lookups=syn.lookups_arrays(c))
    with pytest.raises(_lib.PlonkB200Error, match="zero-knowledge mode does not combine with lookups"):
        prover.set_zk(True)
    with pytest.raises(_lib.PlonkB200Error, match="already set"):
        prover._set_lookup_tagged(qk, qtag, cols, rows)
    with pytest.raises(ValueError, match="sharded prover"):
        parallel.ShardedProver.from_arrays(setup, n, pk, lookups=syn.lookups_arrays(c))
    # the refused calls left the provers usable: the fresh one proves plain, the lookup prover its 1216 bytes
    assert len(fresh.prove_arrays(A, B, C, public)) == 768
    raw = prover.prove_arrays(A, B, C, public)
    vk = setup.verification_key_arrays(n, pk, lookups=syn.lookups_arrays(c))
    assert vk.verify_proof(n, pb.LookupProof.from_bytes(raw), public)
