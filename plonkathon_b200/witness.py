"""What a witness check found (``Prover.check_arrays``, ``Prover.check``): every failing gate, copy constraint, lookup
row and shuffle row, without proving.  The library counts each category exactly and lists its lowest ``limit``
locations (csrc/check.cu); ``WitnessReport`` holds them and renders them with the witness's values."""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

CATEGORIES = ("gate", "copy", "key", "lookup", "shuffle")
WIRE = "abc"


def _int(row: np.ndarray) -> int:
    return int.from_bytes(row.tobytes(), "little")


@dataclass
class WitnessReport:
    """Counts and lowest locations of each category:

    * ``gate``: rows whose gate constraint is not 0 (``gate_rows``);
    * ``copy``: cells c = 3 row + col whose value differs from that of sigma(c), the previous cell of its copy cycle
      (``copy_pairs``: (c, sigma(c)));
    * ``key``: cells whose S entry is not a cell label, or repeats the label of a lower cell -- the key is not a
      permutation and no witness can prove with it (``key_cells``);
    * ``lookup``: rows with q_K = 1 whose (a, b, c[, Q_T]) is not a row of the table (``lookup_rows``);
    * ``shuffle``: rows with q_in or q_out whose (a, b, c) occurs a different number of times among the q_in rows than
      among the q_out rows (``shuffle_rows``).

    ``ok`` is True when every count is 0: then rounds 1 and 2 of a proof pass their checks."""
    gate: int
    copy: int
    key: int
    lookup: int
    shuffle: int
    gate_rows: list
    copy_pairs: list
    key_cells: list
    lookup_rows: list
    shuffle_rows: list
    limit: int
    # what __str__ reads: the wires as (n, 32) uint8 arrays, the shuffle selectors, the variable names of the cells
    _wires: tuple = field(default=None, repr=False, compare=False)
    _shuffle: tuple = field(default=None, repr=False, compare=False)
    _names: object = field(default=None, repr=False, compare=False)

    @classmethod
    def _from_library(cls, counts, lists, limit, wires=None, shuffle=None, names=None):
        counts = [int(x) for x in counts]
        lists = [int(x) for x in lists]
        cut = lambda k, width=1: [x for x in lists[k * limit:(k + width) * limit] if x != 0xffffffff]  # noqa: E731
        copy = cut(1, 2)
        return cls(*counts, cut(0), list(zip(copy[0::2], copy[1::2])), cut(3), cut(4), cut(5), limit,
                   wires, shuffle, names)

    @property
    def ok(self) -> bool:
        return not any(getattr(self, k) for k in CATEGORIES)

    def counts(self) -> dict:
        return {k: getattr(self, k) for k in CATEGORIES}

    def _cell(self, c: int) -> str:
        row, col = divmod(c, 3)
        name = self._names(row, col) if self._names else None
        return "(row %d, %s%s)" % (row, WIRE[col], "" if name is None else ": %s" % name)

    def _value(self, c: int):
        row, col = divmod(c, 3)
        return _int(self._wires[col][row]) if self._wires is not None else "?"

    def _occurrences(self, row: int):
        """how often row's (a, b, c) occurs among the q_in rows and among the q_out rows"""
        a, b, c = self._wires
        same = np.ones(len(a), dtype=bool)
        for w in (a, b, c):
            v = w.view(np.uint64)
            same &= (v == v[row]).all(axis=1)
        q_in, q_out = self._shuffle
        return int(np.count_nonzero(same & q_in)), int(np.count_nonzero(same & q_out))

    def lines(self) -> list:
        out = []
        for r in self.gate_rows:
            out.append("gate: row %d is not satisfied (a = %s, b = %s, c = %s)"
                       % (r, self._value(3 * r), self._value(3 * r + 1), self._value(3 * r + 2)))
        for c, s in self.copy_pairs:
            out.append("copy: cell %s = %s but %s on its cycle = %s"
                       % (self._cell(c), self._value(c), self._cell(s), self._value(s)))
        for c in self.key_cells:
            out.append("key: cell %s: its S entry is not a cell label or repeats a lower cell's; the key is not a "
                       "permutation, so no witness proves with it" % self._cell(c))
        for r in self.lookup_rows:
            out.append("lookup: row %d (a, b, c) = (%s, %s, %s) is not a row of the table"
                       % (r, self._value(3 * r), self._value(3 * r + 1), self._value(3 * r + 2)))
        for r in self.shuffle_rows:
            if self._wires is not None and self._shuffle is not None:
                q_in, q_out = self._shuffle
                side = "q_in and q_out" if q_in[r] and q_out[r] else "q_in" if q_in[r] else "q_out"
                n_in, n_out = self._occurrences(r)
                out.append("shuffle: row %d (%s) tuple occurs %dx in, %dx out" % (r, side, n_in, n_out))
            else:
                out.append("shuffle: row %d tuple occurs a different number of times in and out" % r)
        for k, listed in (("gate", self.gate_rows), ("copy", self.copy_pairs), ("key", self.key_cells),
                          ("lookup", self.lookup_rows), ("shuffle", self.shuffle_rows)):
            if getattr(self, k) > len(listed):
                out.append("%s: %d more" % (k, getattr(self, k) - len(listed)))
        return out

    def __str__(self) -> str:
        if self.ok:
            return "witness satisfies every constraint"
        head = "witness fails: " + ", ".join("%d %s" % (getattr(self, k), k) for k in CATEGORIES if getattr(self, k))
        return "\n".join([head] + ["  " + s for s in self.lines()])
