"""CPU: the independent witness checker (tests/witness_check.py) that the GPU witness check is compared against.

On every proof kind (plain, four custom terms, next-row, shuffle, next-row shuffle, one table, tagged) at n = 16 and 64
its report is empty iff the oracle (tests/extended_oracle.py) proves, for the valid witness and for planted faults; on a
hand-built circuit it gives the known answers; and ``Prover.check_arrays`` refuses malformed inputs before the library
is called."""
import random

import pytest

from oracle import fast as F
from plonkathon_b200 import synthetic as syn
from tests import extended_oracle as XO
from tests import witness_check as WC

R = WC.R
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
NEXT = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
FOUR = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]


def _table(bits, op):
    rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(col) for col in zip(*rows)]


def kind_circuit(kind, log_n, seed=11, n_public=2):
    """a synthetic circuit of a proof kind that uses all of its feature"""
    n = 1 << log_n
    kw = {"plain": {}, "custom": dict(custom=FOUR), "next_row": dict(custom=NEXT), "shuffle": dict(shuffle=True),
          "next_row_shuffle": dict(custom=NEXT, shuffle=True),
          "lookup": dict(lookup=[list(range(n // 2)), [0] * (n // 2), [0] * (n // 2)]),
          "tagged": dict(lookups=[[list(range(4)), [0] * 4, [0] * 4], _table(1, lambda x, y: x ^ y),
                                  _table(1, lambda x, y: x & y)])}[kind]
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, **kw)
        if (all(any(col) for _, col in c.custom) and (not c.shuffle or any(c.shuffle[0]))
                and all(any(q) for q, _ in c.lookups or ([c.lookup] if c.lookup else []))):
            return c
        seed += 1000


KINDS = ["plain", "custom", "next_row", "shuffle", "next_row_shuffle", "lookup", "tagged"]


def faults(c, rng):
    """(name, A, B, C, public) witnesses with one planted fault each, and the valid one first"""
    n = c.group_order
    A, B, C = (list(x) for x in c.wires_values())
    public = c.public_values()
    out = [("valid", A, B, C, public)]
    r = rng.randrange(c.n_public, c.n_constraints)
    out.append(("output", A, B, C[:r] + [(C[r] + 1) % R] + C[r + 1:], public))
    out.append(("public", A, B, C, [(public[0] + 1) % R] + public[1:]))
    # a cell of a variable that appears more than once
    ids = [int(x) for x in c.wire_R[:c.n_constraints]]
    rows = [i for i, v in enumerate(ids) if v >= 0 and (list(c.wire_L).count(v) + list(c.wire_O).count(v)) > 0]
    if rows:
        r = rng.choice(rows)
        out.append(("cycle", A, B[:r] + [(B[r] + 7) % R] + B[r + 1:], C, public))
    # the "no variable" cycle: a cell without a variable holds a value
    empty = [i for i in range(n) if i >= c.n_constraints or int(c.wire_O[i]) < 0]
    if empty:
        r = empty[0]
        out.append(("none", A, B, C[:r] + [5] + C[r + 1:], public))
    qk = None
    if c.lookup:
        qk = c.lookup[0]
    elif c.lookups:
        qk = [max(q[i] for q, _ in c.lookups) for i in range(n)]
    if qk:
        r = rng.choice([i for i in range(n) if qk[i]])
        out.append(("lookup", A[:r] + [(A[r] + 10 ** 6) % R] + A[r + 1:], B, C, public))
    if c.shuffle:
        r = rng.choice([i for i in range(n) if c.shuffle[1][i]])
        out.append(("shuffle", A[:r] + [(A[r] + 3) % R] + A[r + 1:], B, C, public))
    return out


def oracle_proves(c, A, B, C, public) -> bool:
    pk = XO.preprocessed(c)
    try:
        XO.prove(F.Setup(TAU, c.group_order), pk, A, B, C, public, fast=True)
        return True
    except AssertionError:
        return False


@pytest.mark.parametrize("log_n", [4, 6])
@pytest.mark.parametrize("kind", KINDS)
def test_checker_agrees_with_the_oracle(kind, log_n):
    c = kind_circuit(kind, log_n)
    rng = random.Random(log_n * 31 + KINDS.index(kind))
    for name, A, B, C, public in faults(c, rng):
        rep = WC.check_circuit(c, A, B, C, public)
        assert (sum(rep["counts"]) == 0) == oracle_proves(c, A, B, C, public), (name, rep)
        assert (sum(rep["counts"]) == 0) == (name == "valid"), (name, rep)


def _hand_circuit():
    """n = 8: x public; x * y = z; z + x = u; u * u = v; rows 4..7 unused.  Variables 0 x, 1 y, 2 z, 3 u, 4 v."""
    import numpy as np
    n = 8
    L = np.array([0, 0, 2, 3] + [-1] * 4)
    Rw = np.array([-1, 1, 0, 3] + [-1] * 4)
    O_ = np.array([-1, 2, 3, 4] + [-1] * 4)
    QL = [1, 0, 1, 0] + [0] * 4
    QR = [0, 0, 1, 0] + [0] * 4
    QM = [0, 1, 0, 1] + [0] * 4
    QO = [0, R - 1, R - 1, R - 1] + [0] * 4
    x, y = 3, 5
    values = [x, y, x * y, x * y + x, (x * y + x) ** 2]
    return syn.ArrayCircuit(n, 4, L, Rw, O_, QL, QR, QM, QO, [0] * n, 1, values, [])


def test_known_answers_on_a_hand_built_circuit():
    c = _hand_circuit()
    A, B, C = (list(v) for v in c.wires_values())
    public = c.public_values()
    assert WC.check_circuit(c, A, B, C, public)["counts"] == [0, 0, 0, 0, 0]
    # x sits at cells 0 (row 0, a), 3 (row 1, a), 7 (row 2, b): a cycle 0 -> 3 -> 7, sigma = previous cell
    bad = A[:]
    bad[1] = 4  # cell 3: row 1's gate, and the two cells that compare with it
    rep = WC.check_circuit(c, bad, B, C, public)
    assert rep["counts"] == [1, 2, 0, 0, 0]
    assert rep["gate"] == [1] and rep["copy"] == [(3, 0), (7, 3)]
    # a wrong public input: row 0's gate only
    rep = WC.check_circuit(c, A, B, C, [public[0] + 1])
    assert rep["counts"] == [1, 0, 0, 0, 0] and rep["gate"] == [0]
    # the no-variable cycle: an unused cell with a value
    bad = C[:]
    bad[6] = 9
    rep = WC.check_circuit(c, A, B, bad, public)
    assert rep["counts"] == [0, 2, 0, 0, 0] and rep["copy"] == [(20, 19), (21, 20)]  # row 7's a follows it
    # S2 with a non-label and with a duplicated label
    S = [list(s) for s in syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, 8, 4)]
    S2 = S[1][:]
    S2[5] = 12345
    rep = WC.check_circuit(c, A, B, C, public, S=(S[0], S2, S[2]))
    assert rep["counts"][2] == 1 and rep["key"] == [16]
    S2 = S[1][:]
    S2[6] = S[1][5]
    rep = WC.check_circuit(c, A, B, C, public, S=(S[0], S2, S[2]))
    assert rep["key"] == [19]  # row 6, b repeats the label row 5, b names
    # more faults than the limit: counts stay exact
    bad = [(a + 1) % R for a in A]
    rep = WC.check_circuit(c, bad, B, C, public, limit=2)
    full = WC.check_circuit(c, bad, B, C, public, limit=100)
    assert rep["counts"] == full["counts"] and rep["copy"] == full["copy"][:2] and len(full["copy"]) > 2


@pytest.mark.parametrize("kind", ["plain", "next_row_shuffle"])
def test_numpy_copy_failures_equal_the_checker(kind):
    """copy_failures (the 2^24 test's expected copy category) against check on the same changed output wires"""
    import numpy as np
    c = kind_circuit(kind, 8)
    n = c.group_order
    A, B, C = (list(x) for x in c.wires_values())
    changed = np.zeros(3 * n, dtype=bool)
    for r in random.Random(5).sample(range(2, n), 40):
        C[r] ^= 1
        changed[3 * r + 2] = True
    want = WC.check_circuit(c, A, B, C, c.public_values(), limit=3 * n)["copy"]
    got = WC.copy_failures(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints, changed)
    assert [tuple(p) for p in got.tolist()] == want and want


def test_shuffle_counts_a_row_with_both_selectors_on_both_sides():
    n = 4
    Q = {k: [0] * n for k in ("QL", "QR", "QM", "QO", "QC")}
    S = [[pow(5, (R - 1) // n * r, R) * (k + 1) % R for r in range(n)] for k in range(3)]
    A = [1, 2, 2, 3]  # row 0 is on both sides
    rep = WC.check(n, Q, S, A, [0] * n, [0] * n, [], shuffle=([1, 1, 0, 0], [1, 0, 1, 0]))
    assert rep["counts"][4] == 0
    rep = WC.check(n, Q, S, A, [0] * n, [0] * n, [], shuffle=([1, 1, 0, 0], [1, 0, 0, 1]))
    assert rep["shuffle"] == [1, 3]


@pytest.mark.parametrize("args,match", [
    (dict(limit=-1), "limit must be"), (dict(limit=49), "limit must be"), (dict(limit=True), "limit must be"),
    (dict(limit=2.0), "limit must be"), (dict(public=[0] * 17), "17 public inputs for 16 rows"),
    (dict(A=[0] * 17), "A has 17 rows"), (dict(B=__import__("numpy").zeros((16, 31), "uint8")), "B must be an"),
    (dict(C=__import__("numpy").zeros((16, 32), "int64")), "C must be an"), (dict(A=5), "A must be a sequence"),
])
def test_check_arrays_refuses_malformed_inputs_before_the_library(args, match):
    import plonkathon_b200 as pb
    kw = dict(A=[0] * 16, B=[0] * 16, C=[0] * 16, public=[], limit=16)
    kw.update(args)
    p = pb.Prover.__new__(pb.Prover)
    p.group_order = 16  # no library handle: a refusal here never reaches the library
    with pytest.raises(ValueError, match=match):
        p.check_arrays(kw["A"], kw["B"], kw["C"], kw["public"], limit=kw["limit"])


def test_check_needs_a_program():
    import plonkathon_b200 as pb
    p = pb.Prover.__new__(pb.Prover)
    p.program = None
    with pytest.raises(ValueError, match="needs a prover made from a Program"):
        p.check({})


def test_report_text():
    import numpy as np
    import plonkathon_b200 as pb
    n = 64
    wires = tuple(np.zeros((n, 32), np.uint8) for _ in range(3))
    wires[1][17, 0] = 5
    wires[0][9, 0] = 6
    wires[0][40, 0] = 1
    q_in, q_out = np.zeros(n, bool), np.zeros(n, bool)
    q_in[[40, 41]] = True
    wires[0][41, 0] = 1
    q_out[[40, 42]] = True
    limit = 2
    lists = [0xffffffff] * 6 * limit
    lists[2:4] = [3 * 17 + 1, 3 * 9]
    lists[10] = 40
    rep = pb.WitnessReport._from_library([0, 1, 0, 0, 1], lists, limit, wires, (q_in, q_out))
    text = str(rep)
    assert not rep.ok and rep.copy_pairs == [(52, 27)] and rep.shuffle_rows == [40]
    assert "copy: cell (row 17, b) = 5 but (row 9, a) on its cycle = 6" in text
    assert "shuffle: row 40 (q_in and q_out) tuple occurs 2x in, 1x out" in text
    named = pb.WitnessReport._from_library([0, 1, 0, 0, 0], lists, limit, wires, None, lambda r, k: "v%d" % r)
    assert "cell (row 17, b: v17) = 5 but (row 9, a: v9)" in str(named)
    assert str(pb.WitnessReport._from_library([0] * 5, [0xffffffff] * 12, 2)) == "witness satisfies every constraint"
