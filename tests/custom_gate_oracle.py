"""TEST INFRASTRUCTURE ONLY -- the oracle prover and trapdoor verifier with custom gate terms.

The gate constraint gains sum_k Q_k a^i_k b^j_k c^l_k (plonkathon_b200/custom_gates.py).  The reference has no custom
gates, so this extends oracle/plonk_oracle.py in the reference's own structure instead of following a reference file:
one more ``fft_expand`` per term in round 3, and the term's selector weighted by m_k(a_eval, b_eval, c_eval) in
round 5's linearisation.  The restated oracle itself is left as it is (it stays pinned by the reference's fixtures);
``CustomProver`` is a subclass that only adds the custom terms, so a circuit without them takes the pinned code path.
Running it inside ``oracle.fast.c_kernels()`` (``prove(..., fast=True)``) answers its transforms with the C
restatement, as oracle/fast.py does for the plain prover."""
from __future__ import annotations

import dataclasses
from dataclasses import dataclass, field

from oracle import fast as F
from oracle import plonk_oracle as O

R = O.R_MOD


def monomial(exps, a: int, b: int, c: int) -> int:
    i, j, l = exps
    return pow(a, i, R) * pow(b, j, R) % R * pow(c, l, R) % R


@dataclass
class CustomPreprocessed(O.Preprocessed):
    custom: list = field(default_factory=list)  # ((i, j, l), n Lagrange values of Q_k)


class CustomProver(O.Prover):
    """plonk_oracle.Prover with the custom gate terms of ``pk.custom`` added to the gate check, the quotient (round 3)
    and the linearisation (round 5)."""

    def round_1(self, A, B, C):
        if self.check:
            n, pk = self.group_order, self.pk
            A, B, C = ([int(v) % R for v in X] + [0] * (n - len(X)) for X in (A, B, C))
            for i in range(n):
                g = (A[i] * pk.QL[i] + B[i] * pk.QR[i] + A[i] * B[i] * pk.QM[i] + C[i] * pk.QO[i] + self.PI[i] + pk.QC[i]
                     + sum(col[i] * monomial(e, A[i], B[i], C[i]) for e, col in pk.custom))
                assert g % R == 0, "gate %d unsatisfied" % i
        check, self.check = self.check, False  # the plain check would count the custom part as a violation
        try:
            return super().round_1(A, B, C)
        finally:
            self.check = check

    def round_3(self):
        """plonk_oracle.Prover.round_3 with sum_k Q_k(x) m_k(A(x), B(x), C(x)) in the gate term"""
        n, pk = self.group_order, self.pk
        k = self.fft_cofactor
        quarter = O.roots_of_unity(4 * n)
        xs = [k * m % R for m in quarter]
        A_b, B_b, C_b = (self.fft_expand(v) for v in (self.A, self.B, self.C))
        PI_b = self.fft_expand(self.PI)
        QL_b, QR_b, QM_b, QO_b, QC_b = (self.fft_expand(v) for v in (pk.QL, pk.QR, pk.QM, pk.QO, pk.QC))
        QK_b = [(e, self.fft_expand(col)) for e, col in pk.custom]
        Z_b = self.fft_expand(self.Z)
        Zw_b = Z_b[4:] + Z_b[:4]
        S1_b, S2_b, S3_b = (self.fft_expand(v) for v in (pk.S1, pk.S2, pk.S3))
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]
        L0_b = self.fft_expand([1] + [0] * (n - 1))
        al, be, ga = self.alpha, self.beta, self.gamma
        Q = []
        for j in range(4 * n):
            a, b, c, x = A_b[j], B_b[j], C_b[j], xs[j]
            gate = (a * QL_b[j] + b * QR_b[j] + a * b % R * QM_b[j] + c * QO_b[j] + PI_b[j] + QC_b[j]
                    + sum(q[j] * monomial(e, a, b, c) for e, q in QK_b))
            p1 = (a + be * x + ga) * (b + 2 * be * x + ga) % R * (c + 3 * be * x + ga) % R
            p2 = (a + be * S1_b[j] + ga) * (b + be * S2_b[j] + ga) % R * (c + be * S3_b[j] + ga) % R
            num = (gate + al * (p1 * Z_b[j] - p2 * Zw_b[j]) + al * al % R * (Z_b[j] - 1) * L0_b[j]) % R
            Q.append(num * O.inv0(ZH_b[j], R) % R)
        T = self.expanded_evals_to_coeffs(Q)
        assert T[-n:] == [0] * n  # deg T < 3n: degree <= 3 terms keep the quotient in three pieces
        self.T1c, self.T2c, self.T3c = T[:n], T[n:2 * n], T[2 * n:3 * n]
        self.T1, self.T2, self.T3 = O.fft(self.T1c), O.fft(self.T2c), O.fft(self.T3c)
        if self.check:
            assert (O.barycentric_eval(self.T1, k) + O.barycentric_eval(self.T2, k) * pow(k, n, R)
                    + O.barycentric_eval(self.T3, k) * pow(k, 2 * n, R)) % R == Q[0]
        return self.setup.commit(self.T1), self.setup.commit(self.T2), self.setup.commit(self.T3)

    def round_5(self):
        """With the wire values fixed to their evaluations the custom terms are sum_k m_k(a, b, c) Q_k(X): a constant
        selector, so round 5 is plonk_oracle's with QC replaced by QC + sum_k m_k Q_k (fft_expand is linear)."""
        a, b, c = self.a_eval, self.b_eval, self.c_eval
        qc = list(self.pk.QC)
        for e, col in self.pk.custom:
            m = monomial(e, a, b, c)
            qc = [(x + m * y) % R for x, y in zip(qc, col)]
        pk = self.pk
        self.pk = dataclasses.replace(pk, QC=qc)
        try:
            return super().round_5()
        finally:
            self.pk = pk


def prove(setup, pk: CustomPreprocessed, A, B, C, public_inputs, fast: bool = False, check: bool = True) -> dict:
    """oracle proof of a custom-gate circuit; ``fast``: transforms by the C restatement (setup: an oracle.fast.Setup)"""
    if fast:
        with F.c_kernels():
            return CustomProver(setup, pk, check=check).prove(A, B, C, public_inputs)
    return CustomProver(setup, pk, check=check).prove(A, B, C, public_inputs)


def verify_proof_trapdoor(group_order: int, vk: dict, custom_pts, proof: dict, public, tau: int) -> bool:
    """plonk_oracle.verify_proof_trapdoor with the custom terms: the linearisation's gate part gains
    sum_k m_k(a_eval, b_eval, c_eval) [Q_k], which enters exactly like [QC] (weight 1) -- so the plain check runs with
    [QC] + sum_k m_k [Q_k] in QC's place.  custom_pts: ((i, j, l), [Q_k]) in the prover's order."""
    a, b, c = proof["a_eval"], proof["b_eval"], proof["c_eval"]
    qc = O.ec_lincomb_naive([(vk["Qc"], 1)] + [(pt, monomial(e, a, b, c)) for e, pt in custom_pts])
    return O.verify_proof_trapdoor(group_order, dict(vk, Qc=qc), proof, public, tau)


def preprocessed(c, S=None) -> CustomPreprocessed:
    """CustomPreprocessed of a plonkathon_b200.synthetic.ArrayCircuit"""
    from plonkathon_b200 import synthetic as syn
    n = c.group_order
    S1, S2, S3 = S or syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    return CustomPreprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3, list(c.custom))
