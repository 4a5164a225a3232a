"""Wire values of circuits with a shuffle (plonkathon_b200/solve.py ``shuffle=``, csrc/solve.cu
``pb200_solve_wires_shuffle``): a Python restatement of the rule against ``synthetic.memory_circuit``, the witness
checker, the late / clash / order errors, the refusals and the messages; on the GPU the solved wires, their proofs in
plain and zero-knowledge mode, a sort-stress circuit against Python's ``sorted``, the errors, and 2^20 rows."""
import os
import random
from collections import Counter

import numpy as np
import pytest

from plonkathon_b200 import synthetic as syn
from tests import witness_check
from tests.test_solve import SEL, TAU, _ints, _le, _reads_c, restate

R = syn.R
WIRE = "LRO"


# ---- the restatement -------------------------------------------------------------------------------------------------
def restate_shuffle(ids, n, m, sel, custom, inputs, q_in, q_out):
    """-> (A, B, C) as ints or None, unset cells, order (cell, row) pairs, late (cell, row) pairs, clash (cell, reason)
    pairs, under the rule of solve.py's docstring; ids: (n, 3) int array (rows from m on unused)"""
    ids = np.asarray(ids).reshape(n, 3).copy()
    ids[m:] = -1
    if not any(q_out[r] and not q_in[r] for r in range(n)):
        cols, unset, order = restate(ids, n, m, sel, custom, inputs)
        return cols, unset, order, [], []
    ids = ids.tolist()  # ids[r][k]: plain ints, fast to index
    ins = [r for r in range(n) if q_in[r] and not q_out[r]]
    in_set = set(ins)
    outs = [r for r in range(n) if q_out[r] and not q_in[r]]
    p, out_set = outs[0], set(outs)
    defs = {}
    for r in range(m):
        v = int(ids[r][2])
        if r in out_set or v < 0 or sel["QO"][r] == 0 or v in inputs or v in defs:
            continue
        if any(_reads_c(e) and col[r] for e, col in custom):
            continue
        defs[v] = r
    shared = Counter(int(ids[r][k]) for r in outs for k in range(3))
    for r in outs:
        for k in range(3):
            v = int(ids[r][k])
            if v >= 0 and v not in inputs:
                defs[v] = min(defs.get(v, p), p)
    unset, order, late, clash = [], [], [], []
    for c in range(3 * m):
        r, col = divmod(c, 3)
        v = int(ids[r][col])
        if v >= 0 and v not in inputs and v not in defs:
            unset.append(c)
        if col < 2 and r not in out_set and defs.get(int(ids[r][2])) == r and v in defs and defs[v] >= r:
            order.append((c, defs[v]))
    for c in range(3 * n):
        r, col = divmod(c, 3)
        v = int(ids[r][col])
        if r in in_set and v >= 0 and v not in inputs and v in defs and defs[v] >= p:
            late.append((c, defs[v]))
        if r in out_set:
            why = ("no variable" if v < 0 else "input" if v in inputs else "defined" if defs[v] < p
                   else "shared" if shared[v] > 1 else None)
            if why:
                clash.append((c, why))
    if unset or order or late or clash:
        return None, unset, order, late, clash
    val = {-1: 0}
    val.update(inputs)
    for r in range(m + 1):
        if r == p:
            tuples = sorted(tuple(val[int(ids[i][k])] for k in range(3)) for i in ins)
            for o, tup in zip(outs, tuples):
                for k in range(3):
                    val[int(ids[o][k])] = tup[k]
        if r == m:
            break
        v = int(ids[r][2])
        if r in out_set or defs.get(v) != r:
            continue
        a, b = val[int(ids[r][0])], val[int(ids[r][1])]
        s = sel["QL"][r] * a + sel["QR"][r] * b + sel["QM"][r] * a * b + sel["QC"][r]
        for e, col in custom:
            e = tuple(e) + (0,) * (6 - len(e))
            s += col[r] * pow(a, e[0], R) * pow(b, e[1], R) * (0 if any(e[2:]) else 1)
        val[v] = -s * pow(sel["QO"][r], R - 2, R) % R
    cols = [[val[int(ids[r][k])] if r < m else 0 for r in range(n)] for k in range(3)]
    return cols, [], [], [], []


def _ids(c):
    return np.stack([c.wire_L, c.wire_R, c.wire_O], axis=1)


def _sel(c):
    return {k: getattr(c, k) for k in SEL}


def memory_seeds(c, n_addresses):
    """memory_circuit's seeds: x, the addresses, their initial values, the starting time (its first variables)"""
    return {v: c.values[v] for v in range(2 * n_addresses + 2)}


def _restate(c, inputs, shuffle=None):
    q_in, q_out = shuffle or c.shuffle
    return restate_shuffle(_ids(c), c.group_order, c.n_constraints, _sel(c), c.custom, inputs, q_in, q_out)


# ---- CPU -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("log_n,n_addr", [(6, 3), (8, 5)])
def test_restatement_reproduces_memory_circuit_from_its_seeds(log_n, n_addr):
    c = syn.memory_circuit(log_n, n_addr, seed=log_n)
    cols, unset, order, late, clash = _restate(c, memory_seeds(c, n_addr))
    assert (unset, order, late, clash) == ([], [], [], [])
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())
    q_in, q_out = c.shuffle
    assert sum(q_in) == sum(q_out) == (c.group_order - 1) // 5
    outs = [r for r in range(c.group_order) if q_out[r]]
    assert outs == list(range(outs[0], outs[0] + len(outs)))  # one contiguous block
    assert c.n_constraints > outs[-1] + 1  # rows after the sorted block: phase 2 is not empty
    got = witness_check.check_circuit(c, *cols, [])
    assert got["counts"] == [0, 0, 0, 0, 0], got


def test_memory_circuit_addresses_step_by_zero_or_one():
    c = syn.memory_circuit(8, 5, seed=3)
    A = c.wires_values()[0]
    outs = [r for r in range(c.group_order) if c.shuffle[1][r]]
    addrs = [A[r] for r in outs]
    assert addrs[0] == 0 and addrs[-1] == 4 and all(b - a in (0, 1) for a, b in zip(addrs, addrs[1:]))
    # a witness with a gap in the sorted addresses fails the sorted-address gate
    bad = list(A)
    bad[outs[-1]] += 2
    assert witness_check.check_circuit(c, bad, *c.wires_values()[1:], [])["gate"] == [outs[-2]]
    with pytest.raises(ValueError, match="addresses"):
        syn.memory_circuit(4, 4)


def test_build_circuit_shuffle_has_late_in_rows():
    c = syn.build_circuit(8, seed=5, shuffle=True)
    q_in, q_out = c.shuffle
    out_vars = {int(x) for r in range(c.group_order) if q_out[r] for x in _ids(c)[r]}
    from tests.test_solve import free_variables
    inputs = {v: x for v, x in free_variables(c).items() if v not in out_vars}
    cols, unset, order, late, clash = _restate(c, inputs)
    p = q_out.index(1)
    assert late and cols is None and clash == []
    assert all(q_in[cell // 3] and d >= p for cell, d in late)


def _hand(n=16):
    """rows 0-1: two in-rows over inputs 0..5; row 2: gate 6 = 0 + 1; rows 3-4: out-rows over 10..15; row 5: gate
    16 = 10 + 13 (reads out-row variables above p = 3)"""
    ids = np.full((n, 3), -1, np.int64)
    ids[0] = (0, 1, 2)
    ids[1] = (3, 4, 5)
    ids[2] = (0, 1, 6)
    ids[3] = (10, 11, 12)
    ids[4] = (13, 14, 15)
    ids[5] = (10, 13, 16)
    sel = {k: [0] * n for k in SEL}
    for r in (2, 5):
        sel["QL"][r], sel["QR"][r], sel["QO"][r] = R - 1, R - 1, 1
    q_in, q_out = [0] * n, [0] * n
    q_in[0] = q_in[1] = q_out[3] = q_out[4] = 1
    inputs = {0: 7, 1: 2, 2: 9, 3: 5, 4: 1, 5: 3}
    return ids, sel, inputs, q_in, q_out


def test_hand_built_case_and_each_error():
    ids, sel, inputs, q_in, q_out = _hand()
    n = 16
    cols, *errs = restate_shuffle(ids, n, 6, sel, [], inputs, q_in, q_out)
    assert errs == [[], [], [], []]
    assert [cols[k][3] for k in range(3)] == [5, 1, 3] and [cols[k][4] for k in range(3)] == [7, 2, 9]
    assert cols[2][5] == 12
    cases = []
    b = ids.copy()
    b[3, 0] = -1  # no variable (and 16's operand becomes the constant 0)
    cases.append((b, inputs, [(9, "no variable")]))
    cases.append((ids, {**inputs, 11: 4}, [(10, "input")]))
    b = ids.copy()
    b[2, 2] = 12  # row 2 (below p) defines 12
    cases.append((b, inputs, [(11, "defined")]))
    b = ids.copy()
    b[4, 2] = 12  # 12 on two out-row cells
    cases.append((b, inputs, [(11, "shared"), (14, "shared")]))
    for b, ins, want in cases:
        _, unset, order, late, clash = restate_shuffle(b, n, 6, sel, [], ins, q_in, q_out)
        assert clash == want and late == [] and order == []
    # late: the second in-row reads 16, which row 5 (above p) defines, and 12, which the shuffle defines
    b = ids.copy()
    b[1, 1], b[1, 2] = 16, 12
    _, unset, order, late, clash = restate_shuffle(b, n, 6, sel, [], inputs, q_in, q_out)
    assert late == [(4, 5), (5, 3)] and clash == []
    # order naming row p: row 2 (below p) reads out-row variable 13
    b = ids.copy()
    b[2, 1] = 13
    _, unset, order, late, clash = restate_shuffle(b, n, 6, sel, [], inputs, q_in, q_out)
    assert order == [(7, 3)] and late == clash == []
    # a gate row above p with an out-row variable on its O cell only checks it
    b = ids.copy()
    b[5, 2] = 15
    cols, unset, order, late, clash = restate_shuffle(b, n, 6, sel, [], inputs, q_in, q_out)
    assert cols is not None and cols[2][5] == 9


def test_refusals_before_the_library(monkeypatch):
    import plonkathon_b200 as pb
    from plonkathon_b200 import solve as S

    def no_library():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(S, "lib", no_library)
    monkeypatch.setattr(S, "default_context", lambda: None)
    ids, sel, inputs, q_in, q_out = _hand()
    args = (ids[:, 0], ids[:, 1], ids[:, 2], sel, inputs, 16)
    tab = ([0, 1], [0, 1], [0, 1])
    bad = [
        (dict(shuffle=(q_in, q_out), lookup=([0] * 16, tab)), "shuffles do not combine with lookups"),
        (dict(shuffle=(q_in, q_out), lookups=[([0] * 16, tab)]), "shuffles do not combine with lookups"),
        (dict(shuffle=q_in), r"shuffle must be \(q_in, q_out\)"),
        (dict(shuffle=([2] + q_in[1:], q_out)), "q_in must be 0 or 1"),
        (dict(shuffle=(q_in, [R - 1] + q_out[1:])), "q_out must be 0 or 1"),
        (dict(shuffle=(q_in[:-1], q_out)), "q_in has 15 rows"),
        (dict(shuffle=(q_in, [1] + q_out[1:])), "as many q_in rows as q_out rows: 2 and 3"),
    ]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pb.solve_wires(*args, **kw)


def test_late_and_clash_lines():
    from plonkathon_b200.solve import WireSolution
    sol = WireSolution(None, None, None, 0, 0, [], [], 2)
    assert sol.ok and sol.late == sol.clash == 0 and sol.late_cells == sol.clash_cells == []
    ids = np.full(3 * 64, -1, np.int64)
    ids[3 * 40 + 2] = 913
    ids[3 * 31] = 7
    ids[3 * 32 + 1] = 8
    ids[3 * 33 + 2] = 9
    sol = WireSolution(None, None, None, 0, 0, [], [], 4, ids, late=1, clash=5, late_cells=[(3 * 40 + 2, 52)],
                       clash_cells=[(3 * 30, "no variable"), (3 * 31, "input"), (3 * 32 + 1, "defined"),
                                    (3 * 33 + 2, "shared")],
                       _first_out=30, _clash_rows={3 * 32 + 1: 12})
    text = str(sol)
    assert not sol.ok
    assert text.splitlines()[0] == "wires unsolved: 1 late, 5 clash"
    assert ("  late: in-row cell (row 40, O) holds variable 913, which row 52 defines, not before the first out-row 30"
            in text)
    assert "  clash: out-row cell (row 30, L) holds no variable (-1)" in text
    assert "  clash: out-row cell (row 31, L) holds variable 7, an input" in text
    assert "  clash: out-row cell (row 32, R) holds variable 8, which row 12 defines, before the first out-row 30" in text
    assert "  clash: out-row cell (row 33, O) holds variable 9, which another out-row cell holds too" in text
    assert "  clash: 1 more" in text


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _solve(pb, c, inputs, **kw):
    return pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, _sel(c), inputs, c.group_order, n_constraints=c.n_constraints,
                          custom=syn.custom_arrays(c), **kw)


def _prove_both_ways(pb, c, sol, zk=True):
    """the NextRowShuffleProof from the solved device tensors equals the one from the builder's host arrays, and
    verifies; with fixed blinders the zero-knowledge proofs are equal too"""
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n + 9)
    kw = dict(custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))
    prover = pb.Prover.from_arrays(setup, n, pk, **kw)
    assert prover.check_arrays(sol.A, sol.B, sol.C, public).ok
    raw = prover.prove_arrays(sol.A, sol.B, sol.C, public)
    assert raw == prover.prove_arrays(A, B, C, public)
    vk = setup.verification_key_arrays(n, pk, **kw)
    pf = pb.NextRowShuffleProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)
    if zk:
        prover.set_zk_shuffle(True, [(7919 * i + 13) % R for i in range(17)])
        assert prover.prove_arrays(sol.A, sol.B, sol.C, public) == prover.prove_arrays(A, B, C, public)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n,n_addr", [(4, 2), (8, 5), (12, 40), (16, 300)])
def test_gpu_memory_circuit_from_its_seeds(log_n, n_addr):
    import plonkathon_b200 as pb
    c = syn.memory_circuit(log_n, n_addr, seed=log_n)
    seeds = memory_seeds(c, n_addr)
    sol = _solve(pb, c, seeds, device=True, shuffle=syn.shuffle_arrays(c))
    assert sol.ok, str(sol)
    want = c.wires_values()
    for X, w in zip((sol.A, sol.B, sol.C), want):
        assert X.is_cuda and np.array_equal(X.cpu().numpy(), _le(w))
    if log_n <= 12:
        cols = _restate(c, seeds)[0]
        assert tuple(cols) == tuple(list(x) for x in want)
    _prove_both_ways(pb, c, sol, zk=log_n <= 12)
    # without the shuffle the out-row variables are unset
    bare = _solve(pb, c, seeds)
    assert bare.unset > 0 and bare.A is None


def stress_circuit(log_n, seed=7):
    """K = n/4 in-rows over input records, n/4 out-rows of fresh variables right after them, no gates: random field
    elements with duplicate tuples, equal a with different b, equal (a, b) with different c, values near r - 1, and
    words that differ only in the top or only in the bottom 64 bits"""
    n = 1 << log_n
    K = n // 4
    rng = random.Random(seed)
    base = rng.randrange(R - (1 << 64))
    hi = rng.randrange(1 << 60)
    pool = [base, base + 1, base + 2, R - 1, R - 2, hi << 192, (hi + 1) << 192, 0, 1]
    recs = []
    while len(recs) < K:
        kind = rng.randrange(5)
        if kind == 0 and recs:
            recs.append(rng.choice(recs))  # a duplicate
        elif kind == 1 and recs:
            a, b, c = rng.choice(recs)
            recs.append((a, rng.randrange(R), c) if rng.randrange(2) else (a, b, rng.randrange(R)))
        elif kind == 2:
            recs.append(tuple(rng.choice(pool) for _ in range(3)))
        else:
            recs.append(tuple(rng.randrange(R) for _ in range(3)))
    ids = np.full((n, 3), -1, np.int64)
    q_in, q_out = [0] * n, [0] * n
    inputs = {}
    for k, rec in enumerate(recs):
        ids[k] = (3 * k, 3 * k + 1, 3 * k + 2)
        inputs.update({3 * k + j: rec[j] for j in range(3)})
        ids[K + k] = (3 * K + 3 * k, 3 * K + 3 * k + 1, 3 * K + 3 * k + 2)
        q_in[k] = q_out[K + k] = 1
    sel = {k: [0] * n for k in SEL}
    return ids, sel, inputs, q_in, q_out, recs


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [6, 12, 16])
def test_gpu_sort_stress_against_sorted(log_n):
    import plonkathon_b200 as pb
    ids, sel, inputs, q_in, q_out, recs = stress_circuit(log_n)
    n, K = 1 << log_n, len(recs)
    sol = pb.solve_wires(ids[:, 0], ids[:, 1], ids[:, 2], sel, inputs, n, n_constraints=2 * K,
                         shuffle=(q_in, q_out))
    assert sol.ok, str(sol)
    cols = [_ints(X) for X in (sol.A, sol.B, sol.C)]
    got = [tuple(cols[j][K + k] for j in range(3)) for k in range(K)]
    assert got == sorted(recs)  # phase 1 and phase 2 are both empty here
    assert all(cols[j][k] == recs[k][j] for k in range(K) for j in range(3))


@pytest.mark.gpu
def test_gpu_errors_equal_the_restatement():
    import plonkathon_b200 as pb
    ids, sel, inputs, q_in, q_out = _hand()
    n = 16

    def both(b, ins):
        sol = pb.solve_wires(b[:, 0], b[:, 1], b[:, 2], sel, ins, n, n_constraints=6, shuffle=(q_in, q_out), limit=16)
        want = restate_shuffle(b, n, 6, sel, [], ins, q_in, q_out)
        assert (sol.unset_cells, sol.order_cells, sol.late_cells, sol.clash_cells) == tuple(want[1:])
        assert (sol.unset, sol.order, sol.late, sol.clash) == tuple(len(x) for x in want[1:])
        return sol
    sol = both(ids, inputs)
    assert sol.ok and _ints(sol.C)[5] == 12
    b = ids.copy()
    b[3, 0] = -1
    assert both(b, inputs).clash_cells == [(9, "no variable")]
    assert "holds variable 11, an input" in str(both(ids, {**inputs, 11: 4}))
    b = ids.copy()
    b[2, 2] = 12
    assert "which row 2 defines, before the first out-row 3" in str(both(b, inputs))
    b = ids.copy()
    b[4, 2] = 12
    assert both(b, inputs).clash == 2
    b = ids.copy()
    b[1, 1], b[1, 2] = 16, 12
    assert "late: in-row cell (row 1, R) holds variable 16, which row 5 defines" in str(both(b, inputs))
    b = ids.copy()
    b[2, 1] = 13
    assert "order: row 2 reads variable 13 (cell (2, R)), which row 3 defines" in str(both(b, inputs))
    b = ids.copy()
    b[5, 2] = 15
    assert both(b, inputs).ok
    # build_circuit's interleaved out-rows: the late cells the restatement predicts
    c = syn.build_circuit(8, seed=5, shuffle=True)
    out_vars = {int(x) for r in range(c.group_order) if c.shuffle[1][r] for x in _ids(c)[r]}
    from tests.test_solve import free_variables
    ins = {v: x for v, x in free_variables(c).items() if v not in out_vars}
    sol = pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, _sel(c), ins, c.group_order, n_constraints=c.n_constraints,
                         shuffle=syn.shuffle_arrays(c), limit=8)
    want = _restate(c, ins)
    assert (sol.late, sol.clash, sol.unset, sol.order) == (len(want[3]), 0, len(want[1]), len(want[2]))
    assert sol.late_cells == want[3][:8] and sol.late > 0 and sol.A is None
    # the context still solves afterwards
    c = syn.memory_circuit(8, 5, seed=8)
    assert _solve(pb, c, memory_seeds(c, 5), shuffle=syn.shuffle_arrays(c)).ok


@pytest.mark.gpu
def test_gpu_no_out_rows_solves_as_without_a_shuffle():
    import plonkathon_b200 as pb
    from tests.test_solve import free_variables
    c = syn.build_circuit(8, seed=3)
    n = c.group_order
    plain = pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, _sel(c), free_variables(c), n, n_constraints=c.n_constraints)
    for sh in (([0] * n, [0] * n), ([1] * n, [1] * n)):
        got = pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, _sel(c), free_variables(c), n,
                             n_constraints=c.n_constraints, shuffle=sh)
        assert got.ok and all(np.array_equal(x, y) for x, y in zip((got.A, got.B, got.C), (plain.A, plain.B, plain.C)))


def _large(log_n):
    import plonkathon_b200 as pb
    n_addr = 1 << (log_n - 6)
    c = syn.memory_circuit(log_n, n_addr, seed=log_n)
    n = c.group_order
    sol = _solve(pb, c, memory_seeds(c, n_addr), device=True, shuffle=syn.shuffle_arrays(c))
    assert sol.ok, str(sol)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    kw = dict(custom=syn.custom_arrays(c), shuffle=syn.shuffle_arrays(c))
    prover = pb.Prover.from_arrays(setup, n, pk, **kw)
    assert prover.check_arrays(sol.A, sol.B, sol.C, public).ok
    raw = prover.prove_arrays(sol.A, sol.B, sol.C, public)
    assert raw == prover.prove_arrays(A, B, C, public)
    del prover, sol
    vk = setup.verification_key_arrays(n, pk, **kw)
    pf = pb.NextRowShuffleProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_2p20_memory_circuit_from_its_seeds():
    _large(20)


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("PB200_TEST_2P22") != "1", reason="opt-in: PB200_TEST_2P22=1")
def test_gpu_2p22_memory_circuit_from_its_seeds():
    _large(22)
