"""Shuffles: the rows marked by q_in hold the same multiset of (a, b, c) as the rows marked by q_out.

A circuit with a shuffle has two fixed boolean selector columns, q_in and q_out, with as many ones in each.  The claim is
that {(a_i, b_i, c_i) : q_in[i] = 1} and {(a_i, b_i, c_i) : q_out[i] = 1} are equal as multisets: the out-rows are the
in-rows in some order the witness chooses.  No copy constraint joins the two sides, so a circuit can hold a sorted copy
of a list, a memory log in execution order beside the same log sorted by address, or a shuffle of records; next-row
custom gates then state what the sorted side needs ("consecutive rows are ordered", "the same address keeps its value").
A row with both selectors cancels out.

The argument is one more grand product Z3 (DESIGN.md section 1): with challenges theta, kappa drawn after beta, gamma and
w_i = a_i + theta b_i + theta^2 c_i, Z3_(i+1) = Z3_i (1 + q_in[i](kappa + w_i - 1)) / (1 + q_out[i](kappa + w_i - 1)),
and Z3_n = 1.  A shuffle proof has 896 bytes (``ShuffleProof``), 992 with next-row custom gate terms
(``NextRowShuffleProof``).  ``Prover.set_zk_shuffle`` makes the proofs zero-knowledge: A, B, C, Z and the quotient
pieces are blinded as in ``Prover.set_zk``, and Z3 with three more scalars, so a guess at the in-rows or out-rows cannot
be tested against z3_1.  The proof size and the verifier stay the same.

Here: the checks on a shuffle as users give it, ``(q_in, q_out)``, shared by ``Prover.from_arrays``,
``Setup.verification_key_arrays`` and ``synthetic.build_circuit``.  Refused: a shuffle together with lookups, or on the
sharded prover."""
from __future__ import annotations

from .lookup import _column_ints
from .transcript import proof_bytes

PROOF_BYTES = proof_bytes(shuffle=True)
NEXT_ROW_PROOF_BYTES = proof_bytes(next_row=True, shuffle=True)


def check_shuffle(shuffle, group_order: int):
    """``shuffle = (q_in, q_out)`` -> (q_in, q_out) as lists of n ints.  ValueError for a selector that is not n rows
    long or not 0/1 on every row, or for selectors with different numbers of ones."""
    try:
        q_in, q_out = shuffle
    except (TypeError, ValueError):
        raise ValueError("shuffle must be (q_in, q_out)") from None
    out = []
    for name, col in (("q_in", q_in), ("q_out", q_out)):
        col = _column_ints(col)
        if len(col) != group_order:
            raise ValueError("%s has %d rows, expected %d" % (name, len(col), group_order))
        if any(x not in (0, 1) for x in col):
            raise ValueError("%s must be 0 or 1 on every row" % name)
        out.append(col)
    if sum(out[0]) != sum(out[1]):
        raise ValueError("a shuffle needs as many q_in rows as q_out rows: %d and %d" % (sum(out[0]), sum(out[1])))
    return out[0], out[1]


def multisets_match(A, B, C, q_in, q_out) -> bool:
    """whether the in-rows and the out-rows of the wire columns A, B, C (ints) hold the same multiset of (a, b, c)"""
    side = lambda q: sorted((A[i], B[i], C[i]) for i, x in enumerate(q) if x)  # noqa: E731
    return side(q_in) == side(q_out)
