"""Wire values from inputs for circuits with lookups (plonkathon_b200/solve.py ``lookup=`` / ``lookups=``,
csrc/solve.cu): a Python restatement of the rule for rows that define from their table, the shared probe body run on
the CPU (csrc/host_selftest.cpp, hs_solve_lookup), the refusals, and on the GPU: ``synthetic.table_circuit`` solved
from its seeds and proved, the existing lookup kinds solved without their lookup outputs, and the errors."""
import ctypes
import os
import subprocess
import time

import numpy as np
import pytest

from plonkathon_b200 import synthetic as syn
from plonkathon_b200.custom_gates import padded
from plonkathon_b200.lookup import check_lookup, check_lookups, range_table, xor_table
from tests.test_check_host import kind_circuit
from tests.test_solve import SEL, TAU, _ints, _le, free_variables

R = syn.R
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")


# ---- the restatement -------------------------------------------------------------------------------------------------
def _reads_c(e):
    e = padded(e)
    return e[2] > 0 or any(e[3:])


def _table_args(c=None, lookup=None, lookups=None, n=None):
    """-> (q_K, Q_T or None, [t1, t2, t3(, t4)]) as ints, from a circuit or from lookup= / lookups="""
    if c is not None:
        n = c.group_order
        lookup = syn.lookup_arrays(c) if c.lookup else None
        lookups = syn.lookups_arrays(c) if c.lookups else None
    if lookup is not None:
        qk, cols, _ = check_lookup(lookup, n)
        return qk, None, cols
    qk, qt, cols, _ = check_lookups(lookups, n)
    return qk, qt, cols


def restate(ids, n, m, sel, custom, inputs, qk, qt, cols):
    """-> (A, B, C as ints or None, unset cells, order (cell, row) pairs, miss rows, ambiguous rows) under the gate rule
    and the table rule (solve.py's docstring)"""
    ids = np.asarray(ids).reshape(n, 3)
    index = {}
    for r in range(len(cols[0])):
        key = (cols[3][r] if len(cols) > 3 else 0, cols[0][r], cols[1][r])
        index.setdefault(key, set()).add(cols[2][r])
    defs, by_table = {}, set()
    for r in range(m):
        v = int(ids[r, 2])
        if v < 0 or v in inputs or v in defs:
            continue
        gate = sel["QO"][r] != 0 and not any(_reads_c(e) and col[r] for e, col in custom)
        table = sel["QO"][r] == 0 and qk[r] != 0
        if gate or table:
            defs[v] = r
            if table:
                by_table.add(r)
    unset, order = [], []
    for c in range(3 * m):
        v = int(ids[c // 3, c % 3])
        if v >= 0 and v not in inputs and v not in defs:
            unset.append(c)
        r, col = divmod(c, 3)
        if col < 2 and defs.get(int(ids[r, 2])) == r and v in defs and defs[v] >= r:
            order.append((c, defs[v]))
    if unset or order:
        return None, unset, order, [], []
    val = {-1: 0}
    val.update(inputs)
    miss, amb = [], []
    for r in range(m):
        v = int(ids[r, 2])
        if defs.get(v) != r:
            continue
        a, b = val[int(ids[r, 0])], val[int(ids[r, 1])]
        if r in by_table:
            t3 = index.get((qt[r] if qt is not None else 0, a, b), set())
            if len(t3) == 1:
                val[v] = next(iter(t3))
            else:
                (miss if not t3 else amb).append(r)
                val[v] = 0
            continue
        s = sel["QL"][r] * a + sel["QR"][r] * b + sel["QM"][r] * a * b + sel["QC"][r]
        for e, col in custom:
            e = padded(e)
            s += col[r] * pow(a, e[0], R) * pow(b, e[1], R) * (0 if any(e[2:]) else 1)
        val[v] = -s * pow(sel["QO"][r], R - 2, R) % R
    if miss or amb:
        return None, [], [], miss, amb
    return [[val[int(ids[r, k])] if r < m else 0 for r in range(n)] for k in range(3)], [], [], [], []


def _ids(c):
    return np.stack([c.wire_L, c.wire_R, c.wire_O], axis=1)


def _sel(c):
    return {k: getattr(c, k) for k in SEL}


def seeds(c, chains):
    """the free variables of a table circuit: two seeds per chain"""
    return {v: c.values[v] for v in range(2 * chains)}


def reduced_inputs(c):
    """free_variables of a circuit without the O variables of its lookup rows"""
    qk, _, _ = _table_args(c)
    outs = {int(c.wire_O[r]) for r in range(c.n_constraints) if qk[r]}
    return {v: x for v, x in free_variables(c).items() if v not in outs}


def _bits(log_n, tagged):
    """the widest operands whose tables fit 2^log_n rows"""
    return max(b for b in range(1, 5) if (3 if tagged else 1) << (2 * b) <= 1 << log_n)


TABLE_CASES = [(t, w) for t in (False, True) for w in ("deep", "wide")]


def _table_circuit(log_n, tagged, shape):
    chains = 1 if shape == "deep" else max(1, (1 << log_n) // 16)
    return syn.table_circuit(log_n, bits=_bits(log_n, tagged), chains=chains, tagged=tagged, seed=log_n), chains


@pytest.mark.parametrize("tagged,shape", TABLE_CASES)
@pytest.mark.parametrize("log_n", [6, 8])
def test_restatement_reproduces_table_circuit_from_its_seeds(log_n, tagged, shape):
    c, chains = _table_circuit(log_n, tagged, shape)
    assert bool(c.lookups) == tagged and bool(c.lookup) != tagged
    ins = seeds(c, chains)
    assert set(free_variables(c)) - set(ins), "the gate rule alone leaves lookup outputs free"
    cols, unset, order, miss, amb = restate(_ids(c), c.group_order, c.n_constraints, _sel(c), [], ins,
                                            *_table_args(c))
    assert (unset, order, miss, amb) == ([], [], [], [])
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())


@pytest.mark.parametrize("kind", ["lookup", "tagged"])
def test_restatement_reproduces_lookup_kinds_without_their_outputs(kind):
    c = kind_circuit(kind, 6)
    ins = reduced_inputs(c)
    assert len(ins) < len(free_variables(c))
    cols, unset, order, miss, amb = restate(_ids(c), c.group_order, c.n_constraints, _sel(c), c.custom, ins,
                                            *_table_args(c))
    assert (unset, order, miss, amb) == ([], [], [], [])
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())


def _hand(qo_row1=0):
    """n = 8, one XOR table of 2 bits.  Rows: 0: v2 = v0 ^ v1 (lookup); 1: v3 from v2, v0 (lookup, QO = qo_row1, QL = 1);
    2: (v3, -1, -1) lookup with O = -1 (defines nothing); 3: v4 = v2 + v3 (gate)"""
    n = 8
    L = [0, 2, 3, 2] + [-1] * 4
    Rw = [1, 0, -1, 3] + [-1] * 4
    O = [2, 3, -1, 4] + [-1] * 4
    sel = {k: [0] * n for k in SEL}
    sel["QO"][1] = qo_row1
    sel["QL"][1] = 1 if qo_row1 else 0
    sel["QL"][3], sel["QR"][3], sel["QO"][3] = 1, 1, R - 1
    qk = [1, 1, 1, 0] + [0] * 4
    return np.stack([L, Rw, O], axis=1), n, sel, (qk, None, xor_table(2))


def test_restatement_precedence():
    ids, n, sel, tab = _hand()
    cols, *errs = restate(ids, n, 4, sel, [], {0: 1, 1: 3}, *tab)
    assert errs == [[], [], [], []]
    assert [cols[2][r] for r in range(4)] == [2, 3, 0, 5]  # 1^3, 2^1, nothing, 2 + 3
    # a lookup row with QO != 0 keeps the gate rule: QL a + QO c = 0 -> c = -a / QO
    ids, n, sel, tab = _hand(qo_row1=R - 1)
    cols, *errs = restate(ids, n, 4, sel, [], {0: 1, 1: 3}, *tab)
    assert cols[2][1] == 2 and cols[2][3] == 4
    # an input wins over the table: v2 = 1 although 1 ^ 3 = 2, and row 1 reads it
    ids, n, sel, tab = _hand()
    cols, *errs = restate(ids, n, 4, sel, [], {0: 1, 1: 3, 2: 1}, *tab)
    assert errs == [[], [], [], []] and [cols[2][r] for r in range(4)] == [1, 0, 0, 1]
    # an earlier definer wins: a later lookup row whose O variable row 0 already defines only checks
    ids, n, sel, tab = _hand()
    ids = ids.copy()
    ids[3] = [0, 1, 2]
    sel = {k: list(v) for k, v in sel.items()}
    sel["QL"][3] = sel["QR"][3] = 0
    sel["QO"][3] = 0
    tab[0][3] = 1
    cols, *errs = restate(ids, n, 4, sel, [], {0: 1, 1: 3}, *tab)
    assert errs == [[], [], [], []] and cols[2][3] == 2
    # a range row (a, -1, -1) defines nothing: its table row (v, 0, 0) is never read for c
    rt = range_table(4)
    ids = np.array([[0, -1, -1]] + [[-1, -1, -1]] * 7)
    cols, *errs = restate(ids, 8, 1, {k: [0] * 8 for k in SEL}, [], {0: 3}, [1] + [0] * 7, None, rt)
    assert errs == [[], [], [], []] and [cols[k][0] for k in range(3)] == [3, 0, 0]


# ---- the shared probe on the CPU -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hs():
    out = os.path.join(ROOT, "build", "host_selftest_solve_lookup.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    return ctypes.CDLL(out)


def _hs_solve_lookup(hs, ids, n, m, sel, custom, inputs, qk, qt, cols):
    vp = ctypes.c_void_p
    ids = np.ascontiguousarray(np.asarray(ids, np.int64).reshape(-1))
    s = np.concatenate([_le(sel[k]) for k in SEL])
    cust = np.concatenate([_le(col) for _, col in custom]) if custom else np.zeros((1, 32), np.uint8)
    exps = bytes(x for e, _ in custom for x in padded(e)) or b"\0"
    in_ids = np.array(list(inputs), np.int64)
    in_vals = _le(list(inputs.values())) if inputs else np.zeros((1, 32), np.uint8)
    qk_a = _le(qk)
    qt_a = _le(qt) if qt is not None else None
    tab = np.concatenate([_le(col) for col in cols])
    out = np.zeros((3 * n, 32), np.uint8)
    errs = (ctypes.c_uint64 * 2)()
    rc = hs.hs_solve_lookup(ids.ctypes.data_as(vp), n.bit_length() - 1, ctypes.c_uint64(m), s.ctypes.data_as(vp),
                            len(custom), exps, cust.ctypes.data_as(vp), ctypes.c_uint64(len(in_ids)),
                            in_ids.ctypes.data_as(vp), in_vals.ctypes.data_as(vp), qk_a.ctypes.data_as(vp),
                            qt_a.ctypes.data_as(vp) if qt_a is not None else None, tab.ctypes.data_as(vp),
                            ctypes.c_uint64(len(cols[0])), out.ctypes.data_as(vp), errs)
    return rc, [_ints(out[k * n:(k + 1) * n]) for k in range(3)], (errs[0], errs[1])


@pytest.mark.parametrize("tagged,shape", TABLE_CASES)
def test_shared_probe_reproduces_table_circuit(hs, tagged, shape):
    c, chains = _table_circuit(8, tagged, shape)
    rc, cols, errs = _hs_solve_lookup(hs, _ids(c), c.group_order, c.n_constraints, _sel(c), [], seeds(c, chains),
                                      *_table_args(c))
    assert (rc, errs) == (0, (0, 0))
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())


@pytest.mark.parametrize("kind", ["lookup", "tagged"])
def test_shared_probe_reproduces_lookup_kinds(hs, kind):
    c = kind_circuit(kind, 6)
    rc, cols, errs = _hs_solve_lookup(hs, _ids(c), c.group_order, c.n_constraints, _sel(c), c.custom,
                                      reduced_inputs(c), *_table_args(c))
    assert (rc, errs) == (0, (0, 0))
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())


def test_shared_probe_counts_miss_and_ambiguous(hs):
    c, chains = _table_circuit(8, True, "deep")
    ins = seeds(c, chains)
    ins[1] = 1 << _bits(8, True)  # y0 is read once, by the first XOR row: outside the table's domain
    qk, qt, cols = _table_args(c)
    want = restate(_ids(c), c.group_order, c.n_constraints, _sel(c), [], ins, qk, qt, cols)
    assert (want[3], want[4]) == ([0], [])
    rc, _, errs = _hs_solve_lookup(hs, _ids(c), c.group_order, c.n_constraints, _sel(c), [], ins, qk, qt, cols)
    assert (rc, errs) == (2, (1, 0))
    cols = [list(x) for x in cols]
    x0, y0 = c.values[0], c.values[1]
    for w, x in enumerate((x0, y0, (x0 ^ y0) ^ 1, 1)):  # a second t3 for the first XOR row's key
        cols[w].append(x)
    want = restate(_ids(c), c.group_order, c.n_constraints, _sel(c), [], seeds(c, chains), qk, qt, cols)
    rc, _, errs = _hs_solve_lookup(hs, _ids(c), c.group_order, c.n_constraints, _sel(c), [], seeds(c, chains), qk, qt,
                                   cols)
    assert rc == 2 and errs == (len(want[3]), len(want[4])) and want[4]


# ---- refusals and messages -------------------------------------------------------------------------------------------
def test_lookup_refusals_before_the_library(monkeypatch):
    import plonkathon_b200 as pb
    from plonkathon_b200 import solve as S

    def no_library():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(S, "lib", no_library)
    monkeypatch.setattr(S, "default_context", lambda: None)
    c = syn.table_circuit(4, bits=1, tagged=False)
    n = c.group_order
    args = (c.wire_L, c.wire_R, c.wire_O, _sel(c), seeds(c, 1), n)
    qk, tab = syn.lookup_arrays(c)
    bad = [
        (dict(lookup=(qk, tab), lookups=[(qk, tab)]), "not both"),
        (dict(lookup=qk), r"\(q_K, \(t1, t2, t3\)\)"),
        (dict(lookup=([2] + qk[1:], tab)), "q_K must be 0 or 1"),
        (dict(lookup=(qk[:-1], tab)), "q_K has 15 rows"),
        (dict(lookup=(qk, tab[:2])), "exactly three columns"),
        (dict(lookup=(qk, ([], [], []))), "empty"),
        (dict(lookup=(qk, (list(range(17)), [0] * 17, [0] * 17))), "more than the circuit"),
        (dict(lookup=(qk, (tab[0], tab[1], [R] * len(tab[0])))), r"lie in \[0, r\)"),
        (dict(lookups=[]), "at least one table"),
        (dict(lookups=[(qk, tab), (qk, tab)]), "overlap on row"),
        (dict(lookups=[(qk, tab)] * 5), "overlap|more than"),
    ]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            pb.solve_wires(*args, **kw)


def test_miss_and_ambiguous_lines():
    from plonkathon_b200.solve import WireSolution
    sol = WireSolution(None, None, None, 0, 0, [], [], 2)
    assert sol.ok and str(sol) == "wires solved" and sol.miss == 0 and sol.ambiguous_rows == []
    qt = [0] * 64
    qt[40] = 1
    cols = [[0, 2, 2, 3], [0, 2, 2, 16], [0, 0, 4, 19], [0, 0, 0, 1]]
    sol = WireSolution(None, None, None, 0, 0, [], [], 1, None, 3, 1, [40], [41],
                       {40: (3, 17), 41: (2, 2)}, (qt, cols))
    text = str(sol)
    assert not sol.ok
    assert text.splitlines()[0] == "wires unsolved: 3 miss, 1 ambiguous"
    assert "  miss: row 40 looks up (a, b) = (3, 17) in table 1, which has no such row" in text
    assert "  ambiguous: row 41 looks up (a, b) = (2, 2) in table 0, whose rows give c = 0 and c = 4" in text
    assert "  miss: 2 more" in text


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _kw(c):
    return {"lookup": syn.lookup_arrays(c)} if c.lookup else {"lookups": syn.lookups_arrays(c)}


def _solve(pb, c, inputs, **kw):
    return pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, _sel(c), inputs, c.group_order, n_constraints=c.n_constraints,
                          **kw)


def _prove_both_ways(pb, c, sol, zk=True):
    """the proof from the solved device tensors equals the proof from the builder's host arrays, plain and zk"""
    from plonkathon_b200.prover import proof_kind
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    prover = pb.Prover.from_arrays(pb.Setup.generate(TAU, n + 9), n, pk, **_kw(c))
    assert prover.check_arrays(sol.A, sol.B, sol.C, public).ok
    assert prover.prove_arrays(sol.A, sol.B, sol.C, public) == prover.prove_arrays(A, B, C, public)
    if zk:
        k = proof_kind(lookup=True)
        prover.set_zk_lookup(True, [(7919 * i + 13) % R for i in range(k.blinders)])
        assert prover.prove_arrays(sol.A, sol.B, sol.C, public) == prover.prove_arrays(A, B, C, public)


@pytest.mark.gpu
@pytest.mark.parametrize("tagged,shape", TABLE_CASES)
@pytest.mark.parametrize("log_n", [4, 8, 12])
def test_gpu_table_circuit_from_its_seeds(log_n, tagged, shape):
    import plonkathon_b200 as pb
    c, chains = _table_circuit(log_n, tagged, shape)
    sol = _solve(pb, c, seeds(c, chains), device=True, **_kw(c))
    assert sol.ok, str(sol)
    assert str(sol) == "wires solved"
    for X, w in zip((sol.A, sol.B, sol.C), c.wires_values()):
        assert X.is_cuda and np.array_equal(X.cpu().numpy(), _le(w))
    _prove_both_ways(pb, c, sol)


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [8, 12])
@pytest.mark.parametrize("kind", ["lookup", "tagged"])
def test_gpu_lookup_kinds_from_reduced_inputs(kind, log_n):
    import plonkathon_b200 as pb
    c = kind_circuit(kind, log_n)
    sol = _solve(pb, c, reduced_inputs(c), custom=syn.custom_arrays(c), **_kw(c))
    assert sol.ok, str(sol)
    assert [_ints(X) for X in (sol.A, sol.B, sol.C)] == [list(x) for x in c.wires_values()]
    # without the table the lookup outputs are unset
    bare = _solve(pb, c, reduced_inputs(c), custom=syn.custom_arrays(c))
    assert bare.unset > 0 and bare.A is None


def _ok_again(pb):
    """after an error: the context still solves and proves"""
    c, chains = _table_circuit(8, True, "deep")
    sol = _solve(pb, c, seeds(c, chains), device=True, **_kw(c))
    assert sol.ok, str(sol)
    _prove_both_ways(pb, c, sol, zk=False)


@pytest.mark.gpu
def test_gpu_errors_in_a_deep_chain():
    import plonkathon_b200 as pb
    log_n = 12
    bits = _bits(log_n, True)
    c, chains = _table_circuit(log_n, True, "deep")
    ids, sel = _ids(c), _sel(c)
    qk, qt, cols = _table_args(c)
    n, m = c.group_order, c.n_constraints

    # a seed outside the domain: y0 is read once, by row 0 (XOR); every later row depends on it
    ins = seeds(c, chains)
    ins[1] = 1 << bits
    t0 = time.perf_counter()
    sol = _solve(pb, c, ins, **_kw(c))
    took = time.perf_counter() - t0
    assert (sol.unset, sol.order, sol.miss, sol.ambiguous) == (0, 0, 1, 0) and sol.miss_rows == [0]
    assert sol.A is None and not sol.ok and took < 5
    assert "miss: row 0 looks up (a, b) = (%d, %d) in table 1, which has no such row" % (ins[0], 1 << bits) in str(sol)
    _ok_again(pb)

    # a second t3 for one (t1, t2) of the XOR table: every XOR row that reads it is ambiguous
    x0, y0 = c.values[0], c.values[1]
    tabs = [list(map(list, t)) for _, t in syn.lookups_arrays(c)]
    tabs[1][0].append(x0)
    tabs[1][1].append(y0)
    tabs[1][2].append((x0 ^ y0) ^ 1)
    lks = [(q, t) for (q, _), t in zip(syn.lookups_arrays(c), tabs)]
    qk2, qt2, cols2 = check_lookups(lks, n)[:3]
    want = restate(ids, n, m, sel, [], seeds(c, chains), qk2, qt2, cols2)
    sol = _solve(pb, c, seeds(c, chains), lookups=lks, limit=4)
    assert want[4] and want[4][0] == 0
    assert (sol.miss, sol.ambiguous) == (len(want[3]), len(want[4]))
    assert (sol.miss_rows, sol.ambiguous_rows) == (want[3][:4], want[4][:4]) and sol.A is None
    assert ("ambiguous: row 0 looks up (a, b) = (%d, %d) in table 1, whose rows give c = %d and c = %d"
            % (x0, y0, x0 ^ y0, (x0 ^ y0) ^ 1)) in str(sol)
    _ok_again(pb)

    # the tag is part of the key: drop (x0, y0) from the XOR table, keep it in the AND table
    tabs = [list(map(list, t)) for _, t in syn.lookups_arrays(c)]
    k = next(i for i in range(len(tabs[1][0])) if (tabs[1][0][i], tabs[1][1][i]) == (x0, y0))
    for w in range(3):
        del tabs[1][w][k]
    lks = [(q, t) for (q, _), t in zip(syn.lookups_arrays(c), tabs)]
    want = restate(ids, n, m, sel, [], seeds(c, chains), *check_lookups(lks, n)[:3])
    sol = _solve(pb, c, seeds(c, chains), lookups=lks)
    assert sol.miss_rows[:1] == [0] and (sol.miss, sol.ambiguous) == (len(want[3]), len(want[4]))
    assert (sol.miss_rows, sol.ambiguous_rows) == (want[3][:16], want[4][:16])
    _ok_again(pb)

    # order through a lookup row: row 0 (XOR) reads z of the second step, which a later row defines
    bad = ids.copy()
    bad[0, 1] = int(c.wire_O[6])
    sol = pb.solve_wires(bad[:, 0], bad[:, 1], bad[:, 2], sel, seeds(c, chains), n, n_constraints=m, **_kw(c))
    want = restate(bad, n, m, sel, [], seeds(c, chains), qk, qt, cols)
    assert sol.order_cells == want[2][:16] and sol.order == len(want[2]) and (1, 6) in want[2]
    assert (sol.unset, sol.miss, sol.ambiguous) == (len(want[1]), 0, 0) and sol.A is None
    # unset through a lookup row: without seed x0
    ins = seeds(c, chains)
    del ins[0]
    sol = _solve(pb, c, ins, **_kw(c))
    want = restate(ids, n, m, sel, [], ins, qk, qt, cols)
    assert (sol.unset, sol.order, sol.miss) == (len(want[1]), 0, 0) and sol.unset_cells == want[1][:16]
    assert sol.unset_cells[0] == 0
    _ok_again(pb)


@pytest.mark.gpu
def test_gpu_library_refusals():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    c, chains = _table_circuit(4, False, "deep")
    n = c.group_order
    vp = ctypes.c_void_p
    ctx = pb.default_context()
    ids = np.ascontiguousarray(_ids(c).reshape(-1), dtype=np.int64)
    sels = [_le(getattr(c, k)) for k in SEL]
    in_ids = np.array([0, 1], np.int64)
    in_vals = _le([c.values[0], c.values[1]])
    qk, tab = syn.lookup_arrays(c)
    out = [np.zeros((n, 32), np.uint8) for _ in range(3)]
    counts = (ctypes.c_uint64 * 4)()
    lists = (ctypes.c_uint32 * 5)()

    def call(qk_a, t, rows, qt=None, t4=None):
        return _lib.lib().pb200_solve_wires_lookup(
            ctx.handle, ids.ctypes.data_as(vp), 4, c.n_constraints, (vp * 5)(*[s.ctypes.data for s in sels]), 0, b"\0",
            (vp * 1)(), 2, in_ids.ctypes.data_as(vp), in_vals.ctypes.data_as(vp), qk_a.ctypes.data_as(vp),
            qt.ctypes.data_as(vp) if qt is not None else None, *[x.ctypes.data_as(vp) for x in t],
            t4.ctypes.data_as(vp) if t4 is not None else None, rows, 1, counts, lists, None,
            (vp * 3)(*[o.ctypes.data for o in out]), 0)

    t = [_le(x) for x in tab]
    err = lambda: _lib.lib().pb200_last_error().decode()  # noqa: E731
    assert call(_le(qk), t, len(tab[0])) == 0 and counts[:] == [0, 0, 0, 0]
    assert call(_le([2] + list(qk[1:])), t, len(tab[0])) == 1 and "q_K must be 0 or 1" in err()
    assert call(_le(qk), t, 0) == 1 and "empty" in err()
    assert call(_le(qk), [_le(list(range(17)))] * 3, 17) == 1 and "more rows than the circuit" in err()
    assert call(_le(qk), [t[0], t[1], np.full_like(t[2], 255)], len(tab[0])) == 1 and "table value not reduced" in err()
    qt = np.zeros((n, 32), np.uint8)
    qt[np.flatnonzero(np.array(qk) == 0)[0], 0] = 1
    t4 = _le([0] * len(tab[0]))
    assert call(_le(qk), t, len(tab[0]), qt, t4) == 1 and "Q_T must be 0 where q_K = 0" in err()
    assert call(_le(qk), t, len(tab[0]), np.full((n, 32), 255, np.uint8), t4) == 1 and "not reduced" in err()
    assert call(_le(qk), t, len(tab[0]), qt) == 1 and "both Q_T and the table tag column" in err()
    _ok_again(pb)


def _large(log_n, chains):
    import plonkathon_b200 as pb
    c = syn.table_circuit(log_n, chains=chains, seed=log_n)
    n = c.group_order
    sol = _solve(pb, c, seeds(c, chains), device=True, **_kw(c))
    assert sol.ok, str(sol)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk, **_kw(c))
    raw = prover.prove_arrays(sol.A, sol.B, sol.C, public)
    assert raw == prover.prove_arrays(A, B, C, public)
    del prover, sol
    vk = setup.verification_key_arrays(n, pk, **_kw(c))
    pf = pb.LookupProof.from_bytes(raw)
    assert vk.verify_proof(n, pf, public) and vk.verify_proof_unoptimized(n, pf, public)


@pytest.mark.gpu
def test_gpu_2p20_tagged_from_seeds():
    _large(20, 1)


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("PB200_TEST_2P22") != "1", reason="opt-in: PB200_TEST_2P22=1")
@pytest.mark.parametrize("chains", [1, 1 << 16])
def test_gpu_2p22_tagged_from_seeds(chains):
    _large(22, chains)
