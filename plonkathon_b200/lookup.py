"""Lookups: a plookup argument over fixed tables of three columns.

A circuit with lookups has a boolean selector column q_K and a table (t1, t2, t3) of 1..n rows, padded to n rows by
repeating its last row.  A row i with q_K[i] = 1 claims that (a_i, b_i, c_i) is a row of the table; the table's rows
keep the order the user gives them and may repeat.  The argument is plookup (eprint 2020/315) in the cyclic,
alternating-split form of PlonKup (eprint 2022/086); DESIGN.md describes it.  A lookup proof has 13 G1 points and 12
scalars (1216 bytes, ``LookupProof``).

Several tables (``lookups=[(q_0, (t1, t2, t3)), (q_1, ...), ...]``) are told apart by PlonKup's table tag: the tables
are concatenated, a fourth column t4 holds each table row's id (table k has id k) and the selector Q_T the id of the
table each lookup row reads (0 off lookup rows).  A lookup row then matches (a, b, c, Q_T) against (t1, t2, t3, t4),
so it can only match a row of its own table: merging an XOR and an AND table without the tag would let a row meant
for XOR pass with an AND row.

Here: the checks on a lookup argument as users give it, ``(q_K, (t1, t2, t3))`` or a list of them, shared by
``Prover.from_arrays``, ``Setup.verification_key_arrays``, ``synthetic.build_circuit`` and ``solve_wires``, and common
table shapes (``range_table``, ``op_table``, ``xor_table``, ``and_table``).  Out of scope, and
refused: zero knowledge with lookups, the sharded prover, tables wider than three columns."""
from __future__ import annotations

import numpy as np

from .field import CURVE_ORDER
from .transcript import proof_bytes

PROOF_BYTES = proof_bytes(lookup=True)


def _column_ints(col) -> list:
    """a column as Python ints: a list / tuple of ints, or an (m,32) uint8 / (m,8) uint32 little-endian array"""
    if isinstance(col, np.ndarray) and col.dtype != object:
        raw = np.ascontiguousarray(col).view(np.uint8).reshape(-1, 32).tobytes()
        return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]
    return [int(x.n) if hasattr(x, "n") else int(x) for x in col]


def check_lookup(lookup, group_order: int):
    """``lookup = (q_K, (t1, t2, t3))`` -> (q_K as n ints, [t1, t2, t3] as lists of ints, table rows).
    ValueError for a q_K that is not 0/1 or not n rows long, an empty table, a table longer than n, columns of
    unequal length, fewer or more than three columns, or a value >= r."""
    try:
        qk, table = lookup
    except (TypeError, ValueError):
        raise ValueError("lookup must be (q_K, (t1, t2, t3))") from None
    qk = _column_ints(qk)
    if len(qk) != group_order:
        raise ValueError("q_K has %d rows, expected %d" % (len(qk), group_order))
    if any(x not in (0, 1) for x in qk):
        raise ValueError("q_K must be 0 or 1 on every row")
    table = list(table)
    if len(table) != 3:
        raise ValueError("a lookup table has exactly three columns (t1, t2, t3), got %d" % len(table))
    cols = [_column_ints(c) for c in table]
    rows = len(cols[0])
    if any(len(c) != rows for c in cols):
        raise ValueError("lookup table columns of unequal length: %s" % [len(c) for c in cols])
    if rows == 0:
        raise ValueError("the lookup table is empty")
    if rows > group_order:
        raise ValueError("the lookup table has %d rows, more than the circuit's %d" % (rows, group_order))
    if any(not 0 <= x < CURVE_ORDER for c in cols for x in c):
        raise ValueError("lookup table values must lie in [0, r)")
    return qk, cols, rows


def check_lookups(lookups, group_order: int):
    """``lookups = [(q_0, (t1, t2, t3)), (q_1, ...), ...]``, one entry per table -> (q_K, Q_T as n ints each,
    [t1, t2, t3, t4] as lists of ints over the concatenated tables, total rows).  Table k has id k: t4 is k on its rows
    and Q_T is k where q_k = 1.  Each entry is checked as ``check_lookup`` checks ``lookup=``; ValueError also for an
    empty list, selectors that overlap on a row (naming it) and more table rows in all than n."""
    try:
        lookups = list(lookups)
    except TypeError:
        raise ValueError("lookups must be a list of (q_K, (t1, t2, t3)), one per table") from None
    if not lookups:
        raise ValueError("lookups needs at least one table")
    qk, qtag = [0] * group_order, [0] * group_order
    cols, total = [[], [], [], []], 0
    for k, lookup in enumerate(lookups):
        q, tab, rows = check_lookup(lookup, group_order)
        for i in range(group_order):
            if q[i]:
                if qk[i]:
                    raise ValueError("lookup selectors overlap on row %d (tables %d and %d)" % (i, qtag[i], k))
                qk[i], qtag[i] = 1, k
        for w in range(3):
            cols[w] += tab[w]
        cols[3] += [k] * rows
        total += rows
    if total > group_order:
        raise ValueError("the lookup tables have %d rows in all, more than the circuit's %d" % (total, group_order))
    return qk, qtag, cols, total


def padded_table(cols, group_order: int):
    """the columns padded to n rows by repeating their last row"""
    return [c + [c[-1]] * (group_order - len(c)) for c in cols]


def to_le_rows(ints) -> np.ndarray:
    """ints -> contiguous (m,32) uint8 little-endian"""
    raw = b"".join(int(x).to_bytes(32, "little") for x in ints)
    return np.frombuffer(raw, dtype=np.uint8).reshape(-1, 32).copy()


# ---- common table shapes, as (t1, t2, t3) lists of ints ---------------------------------------------------------------
def range_table(k: int):
    """(v, 0, 0) for v < k: a lookup row (a, 0, 0) checks a < k"""
    return [list(range(k)), [0] * k, [0] * k]


def op_table(bits: int, op):
    """(x, y, op(x, y)) for x, y < 2^bits, x-major"""
    rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(c) for c in zip(*rows)]


def xor_table(bits: int):
    """(x, y, x ^ y) for x, y < 2^bits"""
    return op_table(bits, lambda x, y: x ^ y)


def and_table(bits: int):
    """(x, y, x & y) for x, y < 2^bits"""
    return op_table(bits, lambda x, y: x & y)
