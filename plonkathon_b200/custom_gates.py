"""Custom gates: selector columns for degree-2 and degree-3 wire terms.

The gate constraint of a circuit with custom terms is

    QL a + QR b + QM a b + QO c + QC + PI + sum_k Q_k a^i_k b^j_k c^l_k = 0

with at most 4 terms.  A term of total degree <= 3 times its selector has degree <= 4(n - 1), the same bound as the
permutation term of the quotient, so the quotient still splits into three pieces of n coefficients and the proof keeps
its 768-byte form.  Only the circuit (one selector column per term) and the verification key (one commitment per term)
grow.  Here: the checks on the exponent triples and the monomial m_k(a, b, c)."""
from __future__ import annotations

MAX_CUSTOM = 4


def check_exponents(exps) -> tuple:
    """Validate a sequence of exponent triples (i, j, l); returns them as a tuple of int triples.  ValueError for more
    than MAX_CUSTOM terms, a total degree outside 2..3 (degree 1 duplicates QL / QR / QO, degree 4 would need a fourth
    quotient piece), QM's term (1, 1, 0) or a repeated triple."""
    out = []
    for e in exps:
        e = tuple(int(x) for x in e)
        if len(e) != 3 or min(e) < 0:
            raise ValueError("custom gate exponents must be three non-negative integers (i, j, l), got %r" % (e,))
        if not 2 <= sum(e) <= 3:
            raise ValueError("custom gate term %r: total degree must be 2 or 3" % (e,))
        if e == (1, 1, 0):
            raise ValueError("custom gate term (1, 1, 0) duplicates QM")
        if e in out:
            raise ValueError("custom gate term %r given twice" % (e,))
        out.append(e)
    if len(out) > MAX_CUSTOM:
        raise ValueError("at most %d custom gate terms, got %d" % (MAX_CUSTOM, len(out)))
    return tuple(out)


def split_terms(custom, group_order: int):
    """``custom``: a sequence of ``((i, j, l), column)`` with n-row columns -> (exponent triples, columns)."""
    custom = list(custom)
    exps = check_exponents([e for e, _ in custom])
    cols = [col for _, col in custom]
    for e, col in zip(exps, cols):
        if len(col) != group_order:
            raise ValueError("custom selector for %r has %d rows, expected %d" % (e, len(col), group_order))
    return exps, cols


def monomial(exps, a, b, c):
    """a^i b^j c^l for field elements (Scalar or int mod r)"""
    i, j, l = exps
    return a ** i * b ** j * c ** l
