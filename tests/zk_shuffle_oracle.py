"""TEST INFRASTRUCTURE ONLY -- the oracle prover of zero-knowledge shuffle proofs, with explicit blinders.

Zero-knowledge mode (tests/zk_oracle.py, b1..b11; on a next-row circuit tests/next_row_oracle.py, b1..b14) and three more
scalars for the shuffle's grand product, always the last three of the m blinders, Z_H = X^n - 1 (DESIGN.md section 1):
  Z3' = Z3 + (b_(m-2) X^2 + b_(m-1) X + b_m) Z_H,   m = 14, or 17 on a next-row circuit.
Z3 is revealed at zeta w and in the linearisation, so it gets one scalar more than its two points.  Q_in and Q_out are
fixed selectors and stay unblinded.  ``ZkShuffleProver`` subclasses ``shuffle_oracle.ShuffleProver``, which sits on
``NextRowProver`` and already blinds A, B, C, Z and the quotient pieces in coefficient form: it gets b1..b11 and three
zeros (plain or same-row terms) or b1..b14 (next-row terms), and Z3's three are kept apart.  Round 2 blinds Z3c after the
parent builds it; round 3 adds the shuffle terms from the blinded coset values of A, B, C and Z3; rounds 4 and 5 use the
blinded Z3c as they are.  The SRS needs n + 6 powers (n + 9 with next-row terms), and
``shuffle_oracle.verify_proof_trapdoor`` verifies the proofs unchanged.  ``prove(..., fast=True)`` runs inside
``oracle.fast.c_kernels()`` with an ``oracle.fast.Setup``."""
from __future__ import annotations

from oracle import fast as F
from oracle import plonk_oracle as O
from tests import next_row_oracle as NR
from tests import shuffle_oracle as SO
from tests import zk_oracle as ZO

R = O.R_MOD
N_BLINDERS = 14            # plain or same-row terms: b1..b11 as zero-knowledge mode, b12..b14 for Z3
N_NEXT_ROW_BLINDERS = 17   # next-row terms: b1..b14 as zero-knowledge mode on such a circuit, b15..b17 for Z3


def blinder_count(pk) -> int:
    return N_NEXT_ROW_BLINDERS if SO.is_next_row(pk) else N_BLINDERS


class ZkShuffleProver(SO.ShuffleProver):
    """ShuffleProver in zero-knowledge mode: ``blinders`` are b1..b_m, m = blinder_count(pk)"""

    def __init__(self, setup, pk: SO.ShufflePreprocessed, blinders, check: bool = True):
        super().__init__(setup, pk, check=check)
        b = [int(x) % R for x in blinders]
        assert len(b) == blinder_count(pk)
        self.blinders = b[:14] if self.next_row else b[:11] + [0, 0, 0]
        self.z3_blinders = b[-3:]  # b_(m-2), b_(m-1), b_m: the X^2, X and constant coefficients
        self.T = None

    def _z3_blinded(self, coeffs):
        c2, c1, c0 = self.z3_blinders
        return ZO.add_zh_multiple(coeffs, [c0, c1, c2], self.group_order)

    def round_2(self):
        z_1, _ = super().round_2()  # Z', and Z3 with its unblinded coefficients (the Z3_n == 1 check)
        self.Z3c = self._z3_blinded(self.Z3c)
        return z_1, NR._commit(self.setup, self.Z3c)

    def expanded_evals_to_coeffs(self, x):
        out = super().expanded_evals_to_coeffs(x)
        if self._extra is not None:  # the quotient T, kept for the tests
            self.T = out
        return out

    def round_3(self):
        n, pk, b = self.group_order, self.pk, self.blinders
        c2, c1, c0 = self.z3_blinders
        xs = [self.fft_cofactor * m % R for m in O.roots_of_unity(4 * n)]
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]

        def blinded(vals, d2, d1, d0):  # the coset values of vals + (d2 X^2 + d1 X + d0) Z_H (NextRowProver.round_3)
            return [(e + ((d2 * x + d1) * x + d0) * zh) % R for e, x, zh in zip(self.fft_expand(vals), xs, ZH_b)]
        A_b, B_b, C_b = (blinded(v, b[11 + w], b[2 * w], b[2 * w + 1]) for w, v in enumerate((self.A, self.B, self.C)))
        Z3_b = blinded(self.Z3, c2, c1, c0)
        Z3w_b = Z3_b[4:] + Z3_b[:4]  # X -> wX on the 4x finer domain
        QI_b, QO_b = self.fft_expand(pk.q_in), self.fft_expand(pk.q_out)
        L0_b = self.fft_expand([1] + [0] * (n - 1))
        th, al = self.theta, self.alpha
        al3 = pow(al, 3, R)
        al4 = al3 * al % R
        extra = []
        for j in range(4 * n):
            K = (self.kappa + A_b[j] + th * B_b[j] + th * th % R * C_b[j] - 1) % R
            num = (al3 * (Z3w_b[j] * (1 + QO_b[j] * K) - Z3_b[j] * (1 + QI_b[j] * K))
                   + al4 * (Z3_b[j] - 1) * L0_b[j]) % R
            extra.append(num * O.inv0(ZH_b[j], R) % R)
        self._extra = extra
        try:
            return NR.NextRowProver.round_3(self)  # A', B', C', Z' and the pieces T1', T2', T3'
        finally:
            self._extra = None


def prove(setup, pk: SO.ShufflePreprocessed, A, B, C, public_inputs, blinders, fast: bool = False) -> dict:
    """the oracle's zero-knowledge shuffle proof (the dict of shuffle_oracle); ``fast``: transforms by the C restatement
    (setup: an oracle.fast.Setup of at least n + 6 powers, n + 9 with next-row terms)"""
    if fast:
        with F.c_kernels():
            return ZkShuffleProver(setup, pk, blinders).prove(A, B, C, public_inputs)
    return ZkShuffleProver(setup, pk, blinders).prove(A, B, C, public_inputs)
