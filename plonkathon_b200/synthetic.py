"""Array-level circuit construction for sizes the reference's front end cannot reach.

The reference compiler (compiler/program.py, compiler/utils.py:45-47) is O(n^2) and string-based; the
2^20 / 2^22-gate configurations are therefore built directly as arrays with the same conventions:
gate selectors as ``AssemblyEqn.gate()`` produces them (compiler/assembly.py:43-68), the copy-constraint
permutation exactly as ``Program.make_s_polynomials`` builds it (compiler/program.py:70-113: for every
variable, sort its cells by (row, column), and store at each cell the label w^row * column of the previous
cell of the cycle; all unused cells form one more cycle under the ``None`` variable).
tests/test_synthetic_vs_reference.py checks this against the reference compiler on the same wiring."""
from __future__ import annotations

import random
from dataclasses import dataclass, field

import numpy as np

from .field import CURVE_ORDER

R = CURVE_ORDER


@dataclass
class ArrayCircuit:
    group_order: int
    n_constraints: int
    # per-row wire variable ids (-1 == None), rows >= n_constraints are unused
    wire_L: np.ndarray
    wire_R: np.ndarray
    wire_O: np.ndarray
    # selector values per row (Python ints mod r)
    QL: list
    QR: list
    QM: list
    QO: list
    QC: list
    n_public: int
    values: list  # value of every variable id
    text: list  # the same circuit in the reference's constraint language (small sizes only)
    # custom gate terms ((i, j, l), selector values per row), plonkathon_b200/custom_gates.py
    custom: list = field(default_factory=list)
    # lookup argument (q_K per row, (t1, t2, t3)), plonkathon_b200/lookup.py; () without lookups
    lookup: tuple = ()
    # lookups over several tables ((q_k per row, (t1, t2, t3)) per table, table k has id k); () without them
    lookups: tuple = ()
    # shuffle (q_in per row, q_out per row), plonkathon_b200/shuffle.py; () without one
    shuffle: tuple = ()

    def wires_values(self):
        val = self.values
        get = lambda ids: [val[i] if i >= 0 else 0 for i in ids.tolist()]  # noqa: E731
        n, m = self.group_order, self.n_constraints
        pad = [0] * (n - m)
        return get(self.wire_L[:m]) + pad, get(self.wire_R[:m]) + pad, get(self.wire_O[:m]) + pad

    def public_values(self):
        return [self.values[i] for i in self.wire_L[:self.n_public].tolist()]


def roots_of_unity(n: int) -> list:
    w = pow(5, (R - 1) // n, R)
    out, cur = [], 1
    for _ in range(n):
        out.append(cur)
        cur = cur * w % R
    return out


def permutation_polys(wire_L, wire_R, wire_O, group_order: int, n_constraints: int):
    """S1, S2, S3 Lagrange values (lists of ints) -- compiler/program.py:70-113."""
    n = group_order
    roots = roots_of_unity(n)
    ids = np.full((n, 3), -1, dtype=np.int64)
    ids[:n_constraints, 0] = wire_L[:n_constraints]
    ids[:n_constraints, 1] = wire_R[:n_constraints]
    ids[:n_constraints, 2] = wire_O[:n_constraints]
    flat = ids.reshape(-1)  # cell index = row * 3 + (column - 1): already sorted by (row, column)
    order = np.argsort(flat, kind="stable")  # groups cells by variable, keeping (row, column) order
    sorted_ids = flat[order]
    # previous cell within each group (cyclically): S[cell] = label(previous cell of the same variable)
    start = np.ones(len(order), dtype=bool)
    start[1:] = sorted_ids[1:] != sorted_ids[:-1]
    prev = np.empty(len(order), dtype=np.int64)
    prev[1:] = order[:-1]
    group_start_pos = np.flatnonzero(start)
    group_end_pos = np.append(group_start_pos[1:], len(order)) - 1
    prev[group_start_pos] = order[group_end_pos]  # first cell of a cycle points at the last
    S = [[0] * n, [0] * n, [0] * n]
    for cell, pc in zip(order.tolist(), prev.tolist()):
        prow, pcol = divmod(pc, 3)
        row, col = divmod(cell, 3)
        S[col][row] = roots[prow] * (pcol + 1) % R
    return S[0], S[1], S[2]


def build_circuit(log_n: int, seed: int = 20260924, n_public: int = 2, fill: float = 1.0,
                  with_text: bool = False, custom=(), lookup=None, lookups=None, shuffle: bool = False) -> ArrayCircuit:
    """Deterministic synthetic circuit with 2^log_n rows: ``n_public`` public-input rows, then a chain of
    multiplication / addition / add-constant gates whose operands are drawn from recently produced
    variables (so the permutation is non-trivial and the witness values are pseudo-random field elements).

    ``custom``: exponent triples (i, j, l) of custom gate terms; rows using them are mixed into the chain (see
    ``_custom_row``).  Without it the random draws, and so the circuit, are exactly those of a plain circuit.
    A term with six exponents (i, j, l, i', j', l') reads the next row: its row takes three operands on its wires and
    puts a new variable on the next row's L wire, which the next row uses as its first operand (a row whose own output
    goes on L leaves it unused).  So such rows chain without a copy constraint between them.  QC pins the term's value,
    computed once every row is placed; the last row of the chain reads whatever row comes next (row 0 when the chain
    fills the circuit: rows are cyclic).  Not together with lookups.

    ``lookup``: a table ``(t1, t2, t3)``; lookup rows are mixed into the chain as one more kind of row (a quarter of
    the rows without custom terms): the wires take a random table row as three new variables, q_K = 1 and every gate
    selector is 0, and later gates use those variables like any other (copy constraints).  Without it the random
    draws are unchanged.

    ``lookups``: a list of tables ``[(t1, t2, t3), ...]``; as ``lookup``, but each lookup row picks its table at random
    (one more draw, only with two or more tables: ``lookups=[x]`` builds the circuit of ``lookup=x``).

    ``shuffle``: out-rows are mixed into the chain as one more kind of row, a quarter of the rows (one more draw per row,
    only with ``shuffle``): an out-row takes the (a, b, c) of a random earlier row not yet shuffled, as three fresh
    variables with no copy constraint and every selector 0; that row gets q_in = 1, the out-row q_out = 1.  So a quarter
    of the rows are in-rows, a quarter out-rows, and the out-rows hold the in-rows' tuples in a random order.  Without it
    the random draws are unchanged.  Not together with lookups."""
    from .custom_gates import check_exponents, is_next_row
    from .lookup import check_lookup, check_lookups
    custom = check_exponents(custom)
    n = 1 << log_n
    if lookup is not None and lookups is not None:
        raise ValueError("pass either lookup= (one table) or lookups= (several tables), not both")
    if (lookup is not None or lookups is not None) and any(is_next_row(e) for e in custom):
        raise ValueError("lookups do not combine with next-row custom gate terms")
    if shuffle and (lookup is not None or lookups is not None):
        raise ValueError("shuffles do not combine with lookups")
    q_in, q_out = [0] * n, [0] * n
    pool = []        # rows that may still become in-rows
    tables = []  # (columns, rows) per table
    if lookup is not None:
        tables = [check_lookup(([0] * n, lookup), n)[1:]]
    if lookups is not None:
        check_lookups([([0] * n, t) for t in lookups], n)  # each table, and their total size
        tables = [check_lookup(([0] * n, t), n)[1:] for t in lookups]
    QKs = [[0] * n for _ in tables]
    rng = random.Random(seed)
    m = max(n_public + 1, int(n * fill))
    m = min(m, n)
    values = []
    wL = np.full(n, -1, dtype=np.int64)
    wR = np.full(n, -1, dtype=np.int64)
    wO = np.full(n, -1, dtype=np.int64)
    QL, QR, QM, QO, QC = ([0] * n for _ in range(5))
    QK = [[0] * n for _ in custom]
    text = []

    def name(i):
        return "v%d" % i

    # public rows: "x public" -> L = 1, O = 0 (compiler/assembly.py:160-164, 43-68)
    for i in range(n_public):
        values.append(rng.randrange(1, R))
        wL[i] = i
        QL[i] = 1
        if with_text:
            text.append("%s public" % name(i))
    # two private seeds
    for _ in range(2):
        values.append(rng.randrange(1, R))
    window = 64
    row = n_public
    first = True
    carry = None     # the variable a next-row row put on this row's L wire
    pinned = []      # (row, term) of every next-row row, whose QC is set at the end
    while row < m:
        nv = len(values)
        lo = max(0, nv - window)
        ia = rng.randrange(lo, nv)
        ib = rng.randrange(lo, nv)
        if first:  # make sure the private seeds are used so every variable appears in some cell
            ia, ib = n_public, n_public + 1
            first = False
        if carry is not None:
            ia, carry = carry, None
        if shuffle and pool and rng.randrange(4) == 0:  # an out-row: an earlier row's (a, b, c) as fresh variables
            k = rng.randrange(len(pool))
            r = pool[k]
            pool[k] = pool[-1]
            pool.pop()
            values.extend(values[w[r]] for w in (wL, wR, wO))
            wL[row], wR[row], wO[row] = nv, nv + 1, nv + 2
            q_in[r], q_out[row] = 1, 1
            row += 1
            continue
        kind = rng.randrange(3 + len(custom) + bool(tables))
        out = nv
        if tables and kind == 3 + len(custom):  # (a, b, c) = a row of table t, q_t = 1
            t = rng.randrange(len(tables)) if len(tables) > 1 else 0
            table, rows = tables[t]
            r = rng.randrange(rows)
            values.extend(table[w][r] for w in range(3))
            wL[row], wR[row], wO[row] = nv, nv + 1, nv + 2
            QKs[t][row] = 1
        elif kind >= 3 and is_next_row(custom[kind - 3]):  # the term over (a, b, c) and the next row's wires
            ic = rng.randrange(lo, nv)
            k = rng.randrange(0, 1 << 30)
            wL[row], wR[row], wO[row] = ia, ib, ic
            QK[kind - 3][row] = 1
            pinned.append((row, kind - 3))
            if row + 1 < m:
                values.append((values[ia] + k) % R)
                carry = out
        elif kind >= 3:
            ic = rng.randrange(lo, nv)
            k = rng.randrange(0, 1 << 30)
            _custom_row(custom[kind - 3], QK[kind - 3], row, (ia, ib, ic), k, values, (wL, wR, wO), (QL, QO, QC))
        elif kind == 0 or ia == ib:  # c <== a * b : M = -1, O = 1
            values.append(values[ia] * values[ib] % R)
            wL[row], wR[row], wO[row] = ia, ib, out
            QM[row], QO[row] = R - 1, 1
            if with_text:
                text.append("%s <== %s * %s" % (name(out), name(ia), name(ib)))
        elif kind == 1:  # c <== a + b : L = R = -1, O = 1
            values.append((values[ia] + values[ib]) % R)
            wL[row], wR[row], wO[row] = ia, ib, out
            QL[row], QR[row], QO[row] = R - 1, R - 1, 1
            if with_text:
                text.append("%s <== %s + %s" % (name(out), name(ia), name(ib)))
        else:  # c <== a + k : L = -1, C = -k, O = 1
            k = rng.randrange(1, 1 << 30)
            values.append((values[ia] + k) % R)
            # a single-variable expression puts the variable on both input wires (compiler/assembly.py:146-148)
            wL[row], wR[row], wO[row] = ia, ia, out
            QL[row], QC[row], QO[row] = R - 1, (R - k) % R, 1
            if with_text:
                text.append("%s <== %s + %d" % (name(out), name(ia), k))
        if shuffle:
            pool.append(row)
        row += 1
    if pinned:
        from .custom_gates import padded
        cell = lambda ids, r: values[ids[r]] if ids[r] >= 0 else 0  # noqa: E731
        for r, t in pinned:
            r1 = (r + 1) % n
            ws = [cell(w, r) for w in (wL, wR, wO)] + [cell(w, r1) for w in (wL, wR, wO)]
            mon = 1
            for x, e in zip(ws, padded(custom[t])):
                mon = mon * pow(x, e, R) % R
            QC[r] = (R - mon) % R
    lk = (QKs[0], tuple(tables[0][0])) if lookup is not None else ()
    lks = tuple((q, tuple(t)) for q, (t, _) in zip(QKs, tables)) if lookups is not None else ()
    return ArrayCircuit(n, m, wL, wR, wO, QL, QR, QM, QO, QC, n_public, values, text, list(zip(custom, QK)), lk, lks,
                        (q_in, q_out) if shuffle else ())


def table_circuit(log_n: int, bits: int = 4, chains: int = 1, tagged: bool = True, seed: int = 1) -> ArrayCircuit:
    """A bit-manipulation circuit whose table rows read computed values and whose computed values come from tables:
    ``chains`` independent chains, interleaved row by row (1: every row depends on the one before it; many: wide).

    Each chain starts from two seeds x, y < 2^bits, the circuit's only free variables, and repeats a step while the
    circuit has room for one more step of every chain.  With ``tagged`` (three tables: range(2^(2 bits)) as table 0,
    XOR as table 1, AND as table 2, ``lookups=``) a step is six rows:
      z = x ^ y (XOR row), w = x & z (AND row), nz = (2^bits - 1) - z (gate), u = 2^bits w + z (gate, recombination),
      (u, 0, 0) in the range table (a pure check, O = -1), p = u nz (gate); then x, y = nz, w.
    Without it (one XOR table, ``lookup=``) four rows: z = x ^ y, nz = (2^bits - 1) - z, u = 2^bits x + z, p = u nz;
    then x, y = y, nz.  Lookup rows have every gate selector 0.  The values are computed here (``wires_values()``);
    ``solve_wires(..., lookup(s)=)`` finds them from the seeds alone.  ValueError when the tables (3 * 2^(2 bits) or
    2^(2 bits) rows) or one step of every chain do not fit 2^log_n rows."""
    from .lookup import and_table, range_table, xor_table
    n = 1 << log_n
    mask = (1 << bits) - 1
    if bits < 1:
        raise ValueError("bits must be at least 1, got %r" % (bits,))
    tabs = [range_table(1 << (2 * bits)), xor_table(bits), and_table(bits)] if tagged else [xor_table(bits)]
    total = sum(len(t[0]) for t in tabs)
    if total > n:
        raise ValueError("the tables have %d rows in all, more than the circuit's %d" % (total, n))
    per_step = 6 if tagged else 4
    if chains < 1 or per_step * chains > n:
        raise ValueError("%d chains of %d-row steps do not fit %d rows" % (chains, per_step, n))
    steps = n // (per_step * chains)
    m = steps * per_step * chains
    rng = random.Random(seed)
    values = []
    for _ in range(2 * chains):
        values.append(rng.randrange(1 << bits))
    x = list(range(0, 2 * chains, 2))
    y = list(range(1, 2 * chains, 2))
    wL = np.full(n, -1, dtype=np.int64)
    wR = np.full(n, -1, dtype=np.int64)
    wO = np.full(n, -1, dtype=np.int64)
    QL, QR, QM, QO, QC = ([0] * n for _ in range(5))
    Q = [[0] * n for _ in tabs]
    T_RANGE, T_XOR, T_AND = (0, 1, 2) if tagged else (None, 0, None)
    row = 0

    def new(v):
        values.append(v)
        return len(values) - 1

    def put(a, b, o):
        nonlocal row
        wL[row], wR[row], wO[row] = a, b, o
        row += 1
        return row - 1

    val = values.__getitem__
    for _ in range(steps):
        z = [new(val(x[k]) ^ val(y[k])) for k in range(chains)]
        for k in range(chains):
            Q[T_XOR][put(x[k], y[k], z[k])] = 1
        if tagged:
            w = [new(val(x[k]) & val(z[k])) for k in range(chains)]
            for k in range(chains):
                Q[T_AND][put(x[k], z[k], w[k])] = 1
        nz = [new(mask - val(z[k])) for k in range(chains)]
        for k in range(chains):
            r = put(z[k], z[k], nz[k])
            QL[r], QC[r], QO[r] = 1, (R - mask) % R, 1
        hi = w if tagged else x
        u = [new((val(hi[k]) << bits) + val(z[k])) for k in range(chains)]
        for k in range(chains):
            r = put(hi[k], z[k], u[k])
            QL[r], QR[r], QO[r] = 1 << bits, 1, R - 1
        if tagged:
            for k in range(chains):
                Q[T_RANGE][put(u[k], -1, -1)] = 1
        p = [new(val(u[k]) * val(nz[k]) % R) for k in range(chains)]
        for k in range(chains):
            r = put(u[k], nz[k], p[k])
            QM[r], QO[r] = R - 1, 1
        x, y = (nz, w) if tagged else (y, nz)
    assert row == m
    lk = (Q[0], tuple(tabs[0])) if not tagged else ()
    lks = tuple((q, tuple(t)) for q, t in zip(Q, tabs)) if tagged else ()
    return ArrayCircuit(n, m, wL, wR, wO, QL, QR, QM, QO, QC, 0, values, [], [], lk, lks)


def _custom_row(exps, Q, row, operands, k, values, wires, sel):
    """One row using the custom term a^i b^j c^l (selector column Q).  The wires of the monomial take the operands;
    the output goes on the first wire the term does not use:
      * l == 0:          c <== a^i b^j + k        (Q = -1, QO = 1, QC = -k), e.g. c = a^2 b, c = a^3 + k;
      * l > 0, i == 0:   a <== b^j c^l + k        (Q = -1, QL = 1, QC = -k), e.g. a = c^3 + k;
      * i, l > 0:        a^i b^j c^l == its value (Q = 1, QC = -value), e.g. the three-wire constraint a b c = k.
    A wire outside the term and the output carries an operand with a zero selector."""
    i, j, l = exps[:3]  # a six-exponent term here has no next-row exponent
    wL, wR, wO = wires
    QL, QO, QC = sel
    ia, ib, ic = operands
    val = lambda v, e: pow(values[v], e, R)  # noqa: E731
    out = len(values)
    if l == 0:
        values.append((val(ia, i) * val(ib, j) + k) % R)
        wL[row], wR[row], wO[row] = ia, (ib if j else ia), out
        Q[row], QO[row], QC[row] = R - 1, 1, (R - k) % R
    elif i == 0:
        values.append((val(ib, j) * val(ic, l) + k) % R)
        wL[row], wR[row], wO[row] = out, (ib if j else ic), ic
        Q[row], QL[row], QC[row] = R - 1, 1, (R - k) % R
    else:
        prod = val(ia, i) * val(ib, j) * val(ic, l) % R
        wL[row], wR[row], wO[row] = ia, ib, ic
        Q[row], QC[row] = 1, (R - prod) % R
        values.append(prod)  # keeps one new variable per row (unused by any cell)


# the running-sum gate over the next row: bit = a(wX) - 2a and bit (bit - 1) = 0, i.e.
# a'^2 - 4 a a' + 4 a^2 - a' + 2 a = 0  (four custom terms and QL = 2)
RUNNING_SUM_TERMS = ((0, 0, 0, 2, 0, 0), (1, 0, 0, 1, 0, 0), (2, 0, 0, 0, 0, 0), (0, 0, 0, 1, 0, 0))


def range_check_circuit(log_n: int, n_values: int, bits: int = 16, seed: int = 1) -> ArrayCircuit:
    """``n_values`` random values below 2^bits, each range-checked by the running sum over the next row: bits + 1 rows
    per value holding acc_0 = 0, acc_1, ..., acc_bits = the value on the L wire, acc_k+1 = 2 acc_k + (bit k from the
    top), and the running-sum gate (RUNNING_SUM_TERMS) on the first ``bits`` of them.  The value's row carries it on
    all three wires (copies), where later gates would read it.  Row 0 holds the constant 0 (QL a = 0) and every acc_0
    is a copy of it; row 1 holds the constant 1 on all three wires (a + b + a b + c = 4), so that no selector column is
    zero.  The rest of the circuit is unused rows."""
    n = 1 << log_n
    m = 2 + n_values * (bits + 1)
    if m > n:
        raise ValueError("%d values of %d bits need %d rows, the circuit has %d" % (n_values, bits, m, n))
    rng = random.Random(seed)
    wL = np.full(n, -1, dtype=np.int64)
    wR = np.full(n, -1, dtype=np.int64)
    wO = np.full(n, -1, dtype=np.int64)
    QL, QR, QM, QO, QC = ([0] * n for _ in range(5))
    Q = [[0] * n for _ in RUNNING_SUM_TERMS]
    values = [0, 1]
    wL[0], QL[0] = 0, 1
    wL[1] = wR[1] = wO[1] = 1
    QL[1], QR[1], QM[1], QO[1], QC[1] = 1, 1, 1, 1, R - 4
    weights = (1, R - 4, 4, R - 1)  # a'^2, a a', a^2, a'
    row = 2
    for _ in range(n_values):
        x = rng.randrange(1 << bits)
        acc = 0
        wL[row] = 0
        for k in range(bits):
            for q, wgt in zip(Q, weights):
                q[row + k] = wgt
            QL[row + k] = 2
            acc = 2 * acc + ((x >> (bits - 1 - k)) & 1)
            values.append(acc)
            wL[row + k + 1] = len(values) - 1
        wR[row + bits] = wO[row + bits] = wL[row + bits]  # the value on all three wires of its row: B, C are not zero
        row += bits + 1
    return ArrayCircuit(n, m, wL, wR, wO, QL, QR, QM, QO, QC, 0, values, [], list(zip(RUNNING_SUM_TERMS, Q)))


# the sorted-address gate over the next row: consecutive sorted addresses step by 0 or 1, (a' - a)(a' - a - 1) = 0,
# i.e. a'^2 - 2 a a' + a^2 - a' + a = 0  (four custom terms and QL = 1)
SORTED_STEP_TERMS = ((0, 0, 0, 2, 0, 0), (1, 0, 0, 1, 0, 0), (2, 0, 0, 0, 0, 0), (0, 0, 0, 1, 0, 0))


def memory_circuit(log_n: int, n_addresses: int, seed: int = 1) -> ArrayCircuit:
    """A memory-checking circuit: a log of memory records in execution order, the same log sorted by address, and gates
    over the sorted side.  ``shuffle=`` lets ``solve_wires`` find its wires from its seeds alone.

    The seeds (every free variable): a multiplier x, the addresses 0..n_addresses-1, each address's initial value and
    a starting time.  Each of (n - 1) // 5 records is up to three rows: the time counter steps by one (an add-constant
    gate), a write stores prev * x + k at its address (a gate; a read stores nothing and reuses the address's last
    value variable), and a record row (address, time, value), every selector 0, q_in = 1.  The first n_addresses
    records write to every address once, in a random order; the rest pick an address at random and write half the
    time.  A contiguous block of out-rows (q_out = 1) follows, as fresh variables, holding the records sorted by
    (address, time, value), with the sorted-address gate (SORTED_STEP_TERMS, QL = 1) on all but its last row, which
    reads the next row (rows are cyclic).  After it, a running sum of the sorted values reads the out-rows' variables.
    ``values`` is the builder's own witness, the sorted side sorted here.  ValueError when the records do not cover
    the addresses."""
    n = 1 << log_n
    n_rec = (n - 1) // 5
    if not 1 <= n_addresses <= n_rec:
        raise ValueError("n_addresses must be in [1, %d] (one record each at least) for 2^%d rows, got %r"
                         % (n_rec, log_n, n_addresses))
    rng = random.Random(seed)
    values = []
    wL = np.full(n, -1, dtype=np.int64)
    wR = np.full(n, -1, dtype=np.int64)
    wO = np.full(n, -1, dtype=np.int64)
    QL, QR, QM, QO, QC = ([0] * n for _ in range(5))
    Q = [[0] * n for _ in SORTED_STEP_TERMS]
    q_in, q_out = [0] * n, [0] * n
    row = 0

    def new(v):
        values.append(v % R)
        return len(values) - 1

    def put(a, b, o):
        nonlocal row
        wL[row], wR[row], wO[row] = a, b, o
        row += 1
        return row - 1

    x = new(rng.randrange(1, R))
    addr = [new(a) for a in range(n_addresses)]
    last = [new(rng.randrange(R)) for _ in range(n_addresses)]
    t = new(rng.randrange(1 << 20))
    first = list(range(n_addresses))
    rng.shuffle(first)
    records = []
    for i in range(n_rec):
        a = first[i] if i < n_addresses else rng.randrange(n_addresses)
        nt = new(values[t] + 1)  # t <== t + 1 : L = -1, C = -1, O = 1
        r = put(t, t, nt)
        QL[r], QC[r], QO[r] = R - 1, R - 1, 1
        t = nt
        if i < n_addresses or rng.randrange(2):  # v <== prev * x + k : M = -1, C = -k, O = 1
            k = rng.randrange(1, 1 << 30)
            v = new(values[last[a]] * values[x] + k)
            r = put(last[a], x, v)
            QM[r], QC[r], QO[r] = R - 1, (R - k) % R, 1
            last[a] = v
        q_in[put(addr[a], t, last[a])] = 1
        records.append((values[addr[a]], values[t], values[last[a]]))
    records.sort()
    sorted_v = []
    for j, rec in enumerate(records):
        r = put(*(new(w) for w in rec))
        q_out[r] = 1
        sorted_v.append(wO[r])
        if j + 1 < len(records):
            for q, wgt in zip(Q, (1, R - 2, 1, R - 1)):
                q[r] = wgt
            QL[r] = 1
    s = -1
    for v in sorted_v:  # s <== s + v : L = R = -1, O = 1 (the first s is the constant 0)
        ns = new((values[s] if s >= 0 else 0) + values[v])
        r = put(s, v, ns)
        QL[r], QR[r], QO[r] = R - 1, R - 1, 1
        s = ns
    return ArrayCircuit(n, row, wL, wR, wO, QL, QR, QM, QO, QC, 0, values, [], list(zip(SORTED_STEP_TERMS, Q)),
                        shuffle=(q_in, q_out))


def circuit_arrays(c: ArrayCircuit):
    """-> (pk dict of (n,32) uint8 arrays, A, B, C arrays, public list) ready for Prover.from_arrays /
    prove_arrays."""
    S1, S2, S3 = permutation_polys(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
    to_le = lambda ints: np.frombuffer(  # noqa: E731
        b"".join(int(x).to_bytes(32, "little") for x in ints), dtype=np.uint8).reshape(-1, 32).copy()
    pk = {"QM": to_le(c.QM), "QL": to_le(c.QL), "QR": to_le(c.QR), "QO": to_le(c.QO), "QC": to_le(c.QC),
          "S1": to_le(S1), "S2": to_le(S2), "S3": to_le(S3)}
    A, B, C = c.wires_values()
    return pk, to_le(A), to_le(B), to_le(C), c.public_values()


def custom_arrays(c: ArrayCircuit):
    """-> the circuit's custom gate terms as ``((i, j, l), (n,32) uint8 array)``, ready for ``Prover.from_arrays(...,
    custom=)`` and ``Setup.verification_key_arrays(..., custom=)``"""
    return [(e, np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in col), dtype=np.uint8).reshape(-1, 32).copy())
            for e, col in c.custom]


def lookup_arrays(c: ArrayCircuit):
    """-> the circuit's lookup argument ``(q_K, (t1, t2, t3))``, ready for ``Prover.from_arrays(..., lookup=)`` and
    ``Setup.verification_key_arrays(..., lookup=)``"""
    return c.lookup[0], c.lookup[1]


def shuffle_arrays(c: ArrayCircuit):
    """-> the circuit's shuffle ``(q_in, q_out)``, ready for ``Prover.from_arrays(..., shuffle=)`` and
    ``Setup.verification_key_arrays(..., shuffle=)``"""
    return c.shuffle[0], c.shuffle[1]


def lookups_arrays(c: ArrayCircuit):
    """-> the circuit's lookups over several tables ``[(q_0, (t1, t2, t3)), ...]``, ready for
    ``Prover.from_arrays(..., lookups=)`` and ``Setup.verification_key_arrays(..., lookups=)``"""
    return list(c.lookups)
