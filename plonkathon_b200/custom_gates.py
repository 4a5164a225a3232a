"""Custom gates: selector columns for wire terms of degree 2 and 3, and terms that read the next row.

The gate constraint of a circuit with custom terms is

    QL a + QR b + QM a b + QO c + QC + PI + sum_k Q_k a^i_k b^j_k c^l_k a'^i'_k b'^j'_k c'^l'_k = 0

with at most 4 terms, where a' = a(wX), b' = b(wX), c' = c(wX) are the wires of the next row (TurboPLONK; rows are
cyclic, so row n - 1 reads row 0).  A term is given by three exponents (i, j, l), a same-row term, or by six
(i, j, l, i', j', l'); (i, j, l) means (i, j, l, 0, 0, 0).  A term of total degree <= 3 times its selector has degree
<= 4(n - 1), the same bound as the permutation term of the quotient, so the quotient still splits into three pieces of
n coefficients.  Without next-row terms the proof keeps its 768-byte form; with one it gains the three evaluations
a(zeta w), b(zeta w), c(zeta w) (``NextRowProof``, 864 bytes).  Only the circuit (one selector column per term) and the
verification key (one commitment per term) grow.  Here: the checks on the exponents and the monomial m_k."""
from __future__ import annotations

MAX_CUSTOM = 4


def padded(e) -> tuple:
    """an exponent tuple as its six-exponent form (i, j, l, i', j', l')"""
    e = tuple(int(x) for x in e)
    return e + (0,) * (6 - len(e))


def is_next_row(e) -> bool:
    """whether the term reads the next row"""
    return any(padded(e)[3:])


def check_exponents(exps) -> tuple:
    """Validate a sequence of exponent tuples (i, j, l) or (i, j, l, i', j', l'); returns them as a tuple of int
    tuples, each as given.  ValueError for more than MAX_CUSTOM terms, a same-row term of total degree outside 2..3
    (degree 1 duplicates QL / QR / QO, degree 4 would need a fourth quotient piece) or equal to QM's term (1, 1, 0), a
    next-row term of total degree outside 1..3 (no selector reads the next row, so degree 1 is new), or a term given
    twice (a three-exponent term and its padded six-exponent form are the same term)."""
    out = []
    for e in exps:
        e = tuple(int(x) for x in e)
        if len(e) not in (3, 6) or min(e) < 0:
            raise ValueError("custom gate exponents must be three (i, j, l) or six (i, j, l, i', j', l') non-negative "
                             "integers, got %r" % (e,))
        if is_next_row(e):
            if not 1 <= sum(e) <= 3:
                raise ValueError("custom gate term %r: a term over the next row must have total degree 1, 2 or 3"
                                 % (e,))
        else:
            if not 2 <= sum(e) <= 3:
                raise ValueError("custom gate term %r: total degree must be 2 or 3" % (e,))
            if padded(e) == (1, 1, 0, 0, 0, 0):
                raise ValueError("custom gate term (1, 1, 0) duplicates QM")
        if padded(e) in [padded(x) for x in out]:
            raise ValueError("custom gate term %r given twice" % (e,))
        out.append(e)
    if len(out) > MAX_CUSTOM:
        raise ValueError("at most %d custom gate terms, got %d" % (MAX_CUSTOM, len(out)))
    return tuple(out)


def split_terms(custom, group_order: int):
    """``custom``: a sequence of ``((i, j, l), column)`` or ``((i, j, l, i', j', l'), column)`` with n-row columns ->
    (exponent tuples, columns)."""
    custom = list(custom)
    exps = check_exponents([e for e, _ in custom])
    cols = [col for _, col in custom]
    for e, col in zip(exps, cols):
        if len(col) != group_order:
            raise ValueError("custom selector for %r has %d rows, expected %d" % (e, len(col), group_order))
    return exps, cols


def monomial(exps, a, b, c, a_next=None, b_next=None, c_next=None):
    """a^i b^j c^l a'^i' b'^j' c'^l' for field elements (Scalar or int mod r); the next-row values are needed only
    by a term that reads them"""
    m = 1
    for x, e in zip((a, b, c, a_next, b_next, c_next), padded(exps)):
        if e:
            m = x ** e * m
    return m
