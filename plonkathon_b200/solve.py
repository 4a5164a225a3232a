"""A circuit's wire values from the values of its input variables, computed on the GPU (csrc/solve.cu).

``solve_wires`` runs a circuit given as arrays -- the wiring ``permutation_arrays`` takes, the gate selectors, the
custom terms -- the way the reference runs a program (compiler/program.py:161-192): a row r < n_constraints defines
its O variable v when v is not -1, QO[r] != 0, no custom term whose selector is non-zero at r reads c or the next
row, v is not an input and no earlier row defines v; it sets c = -(QL a + QR b + QM a b + QC + sum_k Q_k a^i b^j) / QO.

With ``lookup=`` or ``lookups=`` the gate rule stays exactly as it is.  In addition, a row r < n_constraints defines
its O variable from its table when all of these hold:

* q_K[r] != 0 (with ``lookups=``, the table is the one whose q_k is 1 at r, with its tag k);
* QO[r] = 0 (a row with QO != 0 keeps the gate rule, and its lookup is only checked when proving);
* the O variable is not -1, not an input, and not defined by an earlier row (of either kind).

Such a row sets c = t3 of the table row whose (t1, t2), and tag when tagged, equal (a, b) and the row's tag.  Within a
table, t3 must be a function of (t1, t2); table rows that repeat the same (t1, t2, t3) are fine.  A range table
(v, 0, 0) read as (a, -1, -1) defines nothing, so it stays a pure check.  The ``unset`` and ``order`` errors apply to
table-defining rows exactly as to gate rows: an L or R operand must be the constant 0, an input, or defined by a
strictly earlier row.  Two more error kinds can only be found while the rows are evaluated, so they only arise when
``unset`` and ``order`` are both 0:

* ``miss``: a table-defining row whose (tag, a, b) matches no row of its table;
* ``ambiguous``: a table-defining row whose (tag, a, b) matches table rows with different t3.

Each is an exact count with its lowest ``limit`` rows.  With any error, no wires are returned.

With ``shuffle=(q_in, q_out)`` (as ``Prover.from_arrays`` takes it) the out-rows get their values from the shuffle.
In-rows have q_in = 1 and q_out = 0, out-rows q_out = 1 and q_in = 0; a row with both selectors cancels out in the
argument and is an ordinary row here.  p is the first out-row.  The rule:

1. The shuffle defines every variable on an out-row cell, at row p: after every row below p is evaluated, the
   out-rows, in ascending row order, take the in-rows' tuples in ascending lexicographic order of (a, b, c), compared
   as canonical integers in [0, r), a first.  With a = address, b = time, c = value, that is a memory log sorted by
   address and in time order within each address.  Out-rows define nothing by the gate rule or the table rule.  A
   gate row above p with such a variable on its O cell only checks it.
2. Every in-row cell must be known before p: its variable is -1, an input, or defined by a row below p.  Otherwise
   the cell is ``late`` (also when it holds an out-row variable).
3. Every out-row cell must be able to take the shuffled value.  Otherwise the cell is a ``clash``, for one of these
   reasons: it has no variable (-1), its variable is an input, a gate or table row below p defines it, or the variable
   is on another out-row cell too.
4. ``unset`` and ``order`` keep their meaning, with out-row variables defined at row p: a defining row at or below p
   that reads one is an ``order`` error "row r reads variable v (...), which row p defines".

``late`` and ``clash`` are exact counts with their lowest ``limit`` cells, found before any row is evaluated, like
``unset`` and ``order``.  Without out-rows the solve is the one without ``shuffle=``.  A shuffle does not combine with
lookups.

Every other variable (public inputs, rows whose terms involve c or the next row, hints, lookup rows without a table
argument, and shuffle out-rows without ``shuffle=``) must come as an input.  The wires stay on the device if asked,
for ``Prover.check_arrays`` and ``prove_arrays``."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, field

import numpy as np

from ._lib import check, default_context, lib
from .custom_gates import padded, split_terms
from .field import CURVE_ORDER
from .lookup import check_lookup, check_lookups, to_le_rows
from .shuffle import check_shuffle
from .wiring import MAX_ID, MAX_LOG_N, _wire

WIRE = "LRO"
SEL = ("QL", "QR", "QM", "QO", "QC")
# why an out-row cell cannot take its shuffled value (pb200_solve_wires_shuffle's reason codes 0..3)
CLASH_REASONS = ("no variable", "input", "defined", "shared")


@dataclass
class WireSolution:
    """What ``solve_wires`` found: the wires A, B, C when ``ok``, else the errors, each an exact count and its lowest
    ``limit`` locations:

    * ``unset``: cells whose variable is neither an input nor defined by a row (``unset_cells``: cell = 3 row + col);
    * ``order``: L or R cells of a defining row whose variable that row or a later row defines (``order_cells``:
      (cell, the defining row));
    * ``miss``: rows that define from their table and whose (tag, a, b) matches no table row (``miss_rows``);
    * ``ambiguous``: rows that define from their table and whose (tag, a, b) matches table rows with different t3
      (``ambiguous_rows``);
    * ``late``: in-row cells of a shuffle whose variable is defined at or after the first out-row (``late_cells``:
      (cell, the defining row));
    * ``clash``: out-row cells that cannot take the shuffled value (``clash_cells``: (cell, reason), the reason one of
      ``CLASH_REASONS``)."""
    A: object
    B: object
    C: object
    unset: int
    order: int
    unset_cells: list
    order_cells: list
    limit: int
    _ids: np.ndarray = field(default=None, repr=False, compare=False)
    miss: int = 0
    ambiguous: int = 0
    miss_rows: list = field(default_factory=list)
    ambiguous_rows: list = field(default_factory=list)
    # for the miss and ambiguous lines: {row: (a, b)}, and (Q_T per row or None, [t1, t2, t3(, t4)] as ints)
    _operands: dict = field(default=None, repr=False, compare=False)
    _table: tuple = field(default=None, repr=False, compare=False)
    late: int = 0
    clash: int = 0
    late_cells: list = field(default_factory=list)
    clash_cells: list = field(default_factory=list)
    # for the late and clash lines: the first out-row, and {clash cell: the row below it defining its variable}
    _first_out: int = field(default=None, repr=False, compare=False)
    _clash_rows: dict = field(default=None, repr=False, compare=False)

    @property
    def ok(self) -> bool:
        return not (self.unset or self.order or self.miss or self.ambiguous or self.late or self.clash)

    def _table_of(self, row) -> int:
        qt = self._table[0] if self._table else None
        return int(qt[row]) if qt is not None else 0

    def _t3_values(self, tag, a, b) -> list:
        """the distinct t3 of the table rows with key (tag, a, b), in table order"""
        cols = self._table[1]
        out = []
        for r in range(len(cols[0])):
            if cols[0][r] == a and cols[1][r] == b and (len(cols) < 4 or cols[3][r] == tag) and cols[2][r] not in out:
                out.append(cols[2][r])
        return out

    def lines(self) -> list:
        out = []
        for c in self.unset_cells:
            row, col = divmod(c, 3)
            out.append("unset: cell (row %d, %s) variable %d is neither an input nor defined by a row"
                       % (row, WIRE[col], int(self._ids[c])))
        for c, d in self.order_cells:
            row, col = divmod(c, 3)
            out.append("order: row %d reads variable %d (cell (%d, %s)), which row %d defines"
                       % (row, int(self._ids[c]), row, WIRE[col], d))
        for r in self.miss_rows:
            a, b = self._operands[r]
            out.append("miss: row %d looks up (a, b) = (%d, %d) in table %d, which has no such row"
                       % (r, a, b, self._table_of(r)))
        for r in self.ambiguous_rows:
            a, b = self._operands[r]
            tag = self._table_of(r)
            out.append("ambiguous: row %d looks up (a, b) = (%d, %d) in table %d, whose rows give %s"
                       % (r, a, b, tag, " and ".join("c = %d" % c for c in self._t3_values(tag, a, b)[:2])))
        p = self._first_out
        for c, d in self.late_cells:
            row, col = divmod(c, 3)
            out.append("late: in-row cell (row %d, %s) holds variable %d, which row %d defines, not before the first "
                       "out-row %d" % (row, WIRE[col], int(self._ids[c]), d, p))
        for c, why in self.clash_cells:
            row, col = divmod(c, 3)
            head = "clash: out-row cell (row %d, %s)" % (row, WIRE[col])
            v = int(self._ids[c])
            if why == "no variable":
                out.append(head + " holds no variable (-1)")
            elif why == "input":
                out.append(head + " holds variable %d, an input" % v)
            elif why == "defined":
                out.append(head + " holds variable %d, which row %d defines, before the first out-row %d"
                           % (v, self._clash_rows[c], p))
            else:
                out.append(head + " holds variable %d, which another out-row cell holds too" % v)
        for k, listed in (("unset", self.unset_cells), ("order", self.order_cells), ("miss", self.miss_rows),
                          ("ambiguous", self.ambiguous_rows), ("late", self.late_cells),
                          ("clash", self.clash_cells)):
            if getattr(self, k) > len(listed):
                out.append("%s: %d more" % (k, getattr(self, k) - len(listed)))
        return out

    def __str__(self) -> str:
        if self.ok:
            return "wires solved"
        head = "wires unsolved: " + ", ".join("%d %s" % (getattr(self, k), k)
                                              for k in ("unset", "order", "miss", "ambiguous", "late", "clash")
                                              if getattr(self, k))
        return "\n".join([head] + ["  " + s for s in self.lines()])


def _column(name, col, n) -> np.ndarray:
    """a selector column: n ints or an (n, 32) uint8 array of canonical little-endian values"""
    if isinstance(col, np.ndarray) and col.dtype == np.uint8:
        if col.shape != (n, 32):
            raise ValueError("%s must be an (%d, 32) uint8 array, got %s" % (name, n, col.shape))
        return np.ascontiguousarray(col)
    vals = list(col)
    if len(vals) != n:
        raise ValueError("%s must have group_order = %d values, got %d" % (name, n, len(vals)))
    vals = [int(v.n if hasattr(v, "n") else v) for v in vals]
    if any(not 0 <= v < CURVE_ORDER for v in vals):
        raise ValueError("%s holds a value not reduced below r" % name)
    return np.frombuffer(b"".join(v.to_bytes(32, "little") for v in vals), dtype=np.uint8).reshape(n, 32).copy()


def _le_rows(ints) -> np.ndarray:
    """ints in [0, r) -> contiguous (m, 32) uint8 little-endian; through numpy when they all fit 64 bits (q_K, Q_T and
    small tables), else as lookup.to_le_rows"""
    if not ints or max(ints) >= 1 << 64:
        return to_le_rows(ints)
    out = np.zeros((len(ints), 4), np.uint64)
    out[:, 0] = np.array(ints, dtype=np.uint64)
    return out.view(np.uint8).reshape(-1, 32)


def _inputs(inputs):
    """a dict id -> value, or (ids, (k, 32) uint8 values) -> (int64 ids, (k, 32) uint8 values); ValueError for
    duplicate or out-of-range ids and values not reduced below r"""
    if isinstance(inputs, dict):
        ids = np.fromiter((int(k) for k in inputs), dtype=np.int64, count=len(inputs)) if inputs else \
            np.zeros(0, np.int64)
        vals = [int(v.n if hasattr(v, "n") else v) for v in inputs.values()]
        if any(not 0 <= v < CURVE_ORDER for v in vals):
            bad = next(k for k, v in zip(inputs, vals) if not 0 <= v < CURVE_ORDER)
            raise ValueError("input %d: value not reduced below r" % int(bad))
        raw = np.frombuffer(b"".join(v.to_bytes(32, "little") for v in vals), dtype=np.uint8).reshape(-1, 32)
    else:
        try:
            ids, raw = inputs
        except (TypeError, ValueError):
            raise ValueError("inputs must be a dict id -> value or a pair (ids, (k, 32) uint8 values)") from None
        ids = np.asarray(ids)
        if ids.ndim != 1 or not np.issubdtype(ids.dtype, np.integer):
            raise ValueError("input ids must be a 1-D integer array, got %s %s" % (ids.dtype, ids.shape))
        raw = np.asarray(raw)
        if raw.dtype != np.uint8 or raw.shape != (len(ids), 32):
            raise ValueError("input values must be a (%d, 32) uint8 array, got %s %s" % (len(ids), raw.dtype, raw.shape))
        if len(ids):
            words = np.ascontiguousarray(raw).view("<u8")  # (k, 4) little-endian 64-bit words
            r = [(CURVE_ORDER >> (64 * w)) & (2**64 - 1) for w in range(4)]
            lt = np.zeros(len(ids), bool)
            eq = np.ones(len(ids), bool)
            for w in (3, 2, 1, 0):
                lt |= eq & (words[:, w] < np.uint64(r[w]))
                eq &= words[:, w] == np.uint64(r[w])
            if not lt.all():
                k = int(np.flatnonzero(~lt)[0])
                raise ValueError("input %d (variable %d): value not reduced below r" % (k, int(ids[k])))
    ids = ids.astype(np.int64)
    if len(ids) and (ids.min() < 0 or ids.max() > MAX_ID):
        k = int(np.flatnonzero((ids < 0) | (ids > MAX_ID))[0])
        raise ValueError("input %d: variable id %d is outside [0, 2^32 - 2]" % (k, int(ids[k])))
    s = np.sort(ids)
    dup = np.flatnonzero(s[1:] == s[:-1])
    if len(dup):
        raise ValueError("two inputs name variable %d" % int(s[dup[0]]))
    return np.ascontiguousarray(ids), np.ascontiguousarray(raw, dtype=np.uint8)


def solve_wires(wire_L, wire_R, wire_O, pk: dict, inputs, group_order: int, n_constraints: int | None = None,
                custom=(), device: bool = False, limit: int = 16, ctx=None, lookup=None,
                lookups=None, shuffle=None) -> WireSolution:
    """-> ``WireSolution``: the wire values A, B, C of the circuit, each (n, 32) canonical little-endian, or its
    errors.

    ``wire_L``, ``wire_R``, ``wire_O``: variable ids as ``permutation_arrays`` takes them.  ``pk``: a dict with at least
    QL QR QM QO QC (n ints or (n, 32) uint8 arrays).  ``inputs``: a dict variable id -> value, or a pair (ids,
    (k, 32) uint8 values).  ``custom``: the custom terms as ``Prover.from_arrays(custom=)`` takes them.  ``device``:
    A, B, C as (n, 32) uint8 CUDA tensors on the context's device (no copy to the host), else numpy arrays.
    ``limit``: how many locations of each error kind to list.  ``lookup`` = (q_K, (t1, t2, t3)) or ``lookups`` =
    [(q_0, (t1, t2, t3)), ...], as ``Prover.from_arrays`` takes them: lookup rows then define from their table (the
    module docstring has the rule).  ``shuffle`` = (q_in, q_out), as ``Prover.from_arrays`` takes it: the out-rows
    then take the in-rows' tuples in sorted order (the module docstring has the rule).  Malformed arguments are a ValueError before the library is called; the solve runs
    on the GPU of ``ctx`` (default: the default context)."""
    n = group_order
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 2 or n & (n - 1) or n > 1 << MAX_LOG_N:
        raise ValueError("group_order must be a power of two in [2, 2^%d], got %r" % (MAX_LOG_N, n))
    n = int(n)
    m = n if n_constraints is None else n_constraints
    if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 0 <= m <= n:
        raise ValueError("n_constraints must be an integer in [0, group_order = %d], got %r" % (n, m))
    m = int(m)
    if isinstance(limit, bool) or not isinstance(limit, (int, np.integer)) or not 0 <= limit <= 3 * n:
        raise ValueError("limit must be an integer in [0, 3n = %d], got %r" % (3 * n, limit))
    limit = int(limit)
    ids = np.full((n, 3), -1, dtype=np.int64)
    for col, (name, w) in enumerate((("wire_L", wire_L), ("wire_R", wire_R), ("wire_O", wire_O))):
        ids[:m, col] = _wire(name, w, n, m)
    missing = [k for k in SEL if k not in pk]
    if missing:
        raise ValueError("pk lacks %s" % ", ".join(missing))
    sel = [_column(k, pk[k], n) for k in SEL]
    exps, ccols = split_terms(custom, n)
    cust = [_column("custom selector %r" % (e,), c, n) for e, c in zip(exps, ccols)]
    in_ids, in_vals = _inputs(inputs)
    if lookup is not None and lookups is not None:
        raise ValueError("pass either lookup= (one table) or lookups= (several tables), not both")
    table = None
    if lookup is not None:
        qk, tcols, rows = check_lookup(lookup, n)
        table = (qk, None, tcols, rows)
    elif lookups is not None:
        table = check_lookups(lookups, n)
    sh = None
    if shuffle is not None:
        if table is not None:
            raise ValueError("shuffles do not combine with lookups")
        q_in, q_out = check_shuffle(shuffle, n)
        sh = [_le_rows(q) for q in (q_in, q_out)]
    ctx = ctx or default_context()

    vp = ctypes.c_void_p
    sel_arr = (vp * 5)(*[s.ctypes.data for s in sel])
    cust_arr = (vp * max(1, len(cust)))(*[c.ctypes.data for c in cust])
    ebytes = bytes(x for e in exps for x in padded(e)) or b"\0"
    if device:
        import torch
        dev = torch.device("cuda", ctx.device)
        torch.cuda.current_stream(dev).synchronize()  # the blocks may have served work still queued on torch's stream
        out = [torch.empty((n, 32), dtype=torch.uint8, device=dev) for _ in range(3)]
        ptrs = [t.data_ptr() for t in out]
    else:
        out = [np.empty((n, 32), dtype=np.uint8) for _ in range(3)]
        ptrs = [a.ctypes.data for a in out]
    # the mode's entry point, its own arguments, and the entries per listed location of each error kind
    col = lambda a: a.ctypes.data_as(vp) if a is not None else None  # noqa: E731
    extra = ()
    if sh is not None:
        call, args, arity = lib().pb200_solve_wires_shuffle, (col(sh[0]), col(sh[1])), (1, 2, 2, 3)
    elif table is None:
        call, args, arity = lib().pb200_solve_wires, (), (1, 2)
    else:
        qk, qt, tcols, rows = table
        tab = [_le_rows(c) for c in tcols]  # t1 t2 t3, and t4 with lookups=
        args = (col(_le_rows(qk)), col(_le_rows(qt) if qt is not None else None), col(tab[0]), col(tab[1]),
                col(tab[2]), col(tab[3]) if len(tab) > 3 else None, rows)
        call, arity = lib().pb200_solve_wires_lookup, (1, 2, 1, 1)
        operands = np.zeros((max(1, 4 * limit), 32), np.uint8)
        extra = (operands.ctypes.data_as(vp),)
    counts = (ctypes.c_uint64 * len(arity))()
    lists = (ctypes.c_uint32 * max(1, sum(arity) * limit))()
    check(call(ctx.handle, ids.ctypes.data_as(vp), n.bit_length() - 1, m, sel_arr, len(exps), ebytes, cust_arr,
               len(in_ids), in_ids.ctypes.data_as(vp), in_vals.ctypes.data_as(vp), *args, limit, counts, lists, *extra,
               (vp * 3)(*ptrs), 1 if device else 0))
    # each kind's `limit` slots of `a` entries, a used slot's first entry not 0xffffffff
    raw = [int(x) for x in lists[:sum(arity) * limit]]
    listed, at = [], 0
    for a in arity:
        slots = [tuple(raw[at + a * k:at + a * k + a]) for k in range(limit)]
        listed.append([e[0] if a == 1 else e for e in slots if e[0] != 0xffffffff])
        at += a * limit
    ok = not any(counts)
    A, B, C = out if ok else (None, None, None)
    sol = WireSolution(A, B, C, int(counts[0]), int(counts[1]), listed[0], listed[1], limit, ids.reshape(-1))
    if table is not None:
        sol.miss, sol.ambiguous = int(counts[2]), int(counts[3])
        sol.miss_rows, sol.ambiguous_rows = listed[2], listed[3]
        ops = operands.reshape(-1, 32).tobytes()
        val = lambda k: int.from_bytes(ops[32 * k:32 * k + 32], "little")  # noqa: E731
        sol._operands = {r: (val(2 * k), val(2 * k + 1)) for k, r in enumerate(sol.miss_rows)}
        sol._operands.update({r: (val(2 * limit + 2 * k), val(2 * limit + 2 * k + 1))
                              for k, r in enumerate(sol.ambiguous_rows)})
        sol._table = (table[1], table[2])
    if sh is not None:
        sol.late, sol.clash = int(counts[2]), int(counts[3])
        sol.late_cells = listed[2]
        sol.clash_cells = [(c, CLASH_REASONS[why]) for c, why, _ in listed[3]]
        sol._clash_rows = {c: d for c, _, d in listed[3]}
        sol._first_out = next((r for r in range(n) if q_out[r] and not q_in[r]), None)
    return sol
