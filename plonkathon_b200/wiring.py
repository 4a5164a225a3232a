"""The copy-constraint permutation of a circuit's wiring, built on the GPU (csrc/permutation.cu).

A circuit described as wires -- a variable id on each of the 3n cells (L, R, O of every row), -1 where a cell carries
no variable -- needs the permutation columns S1, S2, S3 before it can be proved.  ``permutation_arrays`` computes them
exactly as the reference compiler does (compiler/program.py:70-113; ``synthetic.permutation_polys`` is the CPU
restatement): the cells of one variable form a cycle in (row, column) order, every cell stores the label
omega^row (column + 1) of the previous cell of its cycle, the first cell that of the last, and all unused cells form
one more cycle."""
from __future__ import annotations

import ctypes

import numpy as np

from ._lib import check, default_context, lib

MAX_ID = (1 << 32) - 2  # id + 1 takes the top 32 bits of the 64-bit sort key (with the cell index below it)
MAX_LOG_N = 26          # the prover's range


def _wire(name, w, n, m):
    a = np.asarray(w)
    if a.ndim != 1 or len(a) not in (m, n):
        raise ValueError("%s must be a 1-D array of n_constraints = %d or group_order = %d ids, got shape %s"
                         % (name, m, n, a.shape))
    if not np.issubdtype(a.dtype, np.integer):
        raise ValueError("%s must hold integer variable ids (-1 for no variable), got dtype %s" % (name, a.dtype))
    a = a[:m]
    if len(a) and (a.min() < -1 or a.max() > MAX_ID):
        r = int(np.flatnonzero((a < -1) | (a > MAX_ID))[0])
        raise ValueError("%s[%d] = %d: a variable id must be -1 (no variable) or in [0, 2^32 - 2]" % (name, r, int(a[r])))
    return a


def permutation_arrays(wire_L, wire_R, wire_O, group_order: int, n_constraints: int | None = None, ctx=None) -> dict:
    """-> {"S1", "S2", "S3"}: (n, 32) uint8 arrays of canonical little-endian values, ready to merge into the
    ``pk_arrays`` of ``Prover.from_arrays`` and ``Setup.verification_key_arrays``.

    ``wire_L``, ``wire_R``, ``wire_O``: integer arrays of ``n_constraints`` or ``group_order`` variable ids, -1 for no
    variable, each id in [-1, 2^32 - 2].  Rows from ``n_constraints`` on (default: ``group_order``) are unused: their
    cells are -1 whatever the arrays hold there.  Every input is checked here, before the library is called; the
    permutation itself runs on the GPU of ``ctx`` (default: the default context), with no CPU fallback."""
    n = group_order
    if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 2 or n & (n - 1) or n > 1 << MAX_LOG_N:
        raise ValueError("group_order must be a power of two in [2, 2^%d], got %r" % (MAX_LOG_N, n))
    n = int(n)
    m = n if n_constraints is None else n_constraints
    if isinstance(m, bool) or not isinstance(m, (int, np.integer)) or not 0 <= m <= n:
        raise ValueError("n_constraints must be an integer in [0, group_order = %d], got %r" % (n, m))
    m = int(m)
    ids = np.full((n, 3), -1, dtype=np.int64)
    for col, (name, w) in enumerate((("wire_L", wire_L), ("wire_R", wire_R), ("wire_O", wire_O))):
        ids[:m, col] = _wire(name, w, n, m)
    ctx = ctx or default_context()
    out = np.empty((3, n, 32), dtype=np.uint8)
    check(lib().pb200_permutation(ctx.handle, ids.ctypes.data_as(ctypes.c_void_p), n.bit_length() - 1,
                                  out.ctypes.data_as(ctypes.c_void_p)))
    return {"S1": out[0], "S2": out[1], "S3": out[2]}
