"""TEST INFRASTRUCTURE ONLY -- the oracle prover of zero-knowledge lookup proofs, with explicit blinders.

Plain zero-knowledge mode (tests/zk_oracle.py, b1..b11 = blinders[0..10]) and ten more scalars for the lookup
polynomials the proof commits to, b12..b21 = blinders[11..20], Z_H = X^n - 1 (DESIGN.md section 1):
  F' = F + (b12 X + b13) Z_H,  H1' = H1 + (b14 X^2 + b15 X + b16) Z_H,  H2' = H2 + (b17 X + b18) Z_H,
  Z2' = Z2 + (b19 X^2 + b20 X + b21) Z_H.
T, q_K, Q_T and the table columns are fixed or public and stay unblinded.  ``ZkLookupMixin`` goes in front of
``tagged_lookup_oracle.TaggedProver`` (one table is the case Q_T = t4 = 0), which stays as it is.  Rounds 1 and 2 and the
plain evaluations come from ``zk_oracle.ZkMixin``; step 1L and Z2 run the parent's code behind ``_NoCommit`` (the table
index, the witness checks, the grand product) and commit the blinded polynomials in monomial form; round 3 adds the Z_H
multiples on the coset; round 4 corrects f, h2, h1(zeta w) and z2(zeta w); round 5 builds the linearisation and the two
openings in coefficient form, as ``ZkMixin.round_5`` does.  The SRS needs n + 6 powers.  ``prove(..., fast=True)`` runs
inside ``oracle.fast.c_kernels()`` with an ``oracle.fast.Setup``."""
from __future__ import annotations

from oracle import fast as F
from oracle import plonk_oracle as O
from tests import custom_gate_oracle as CG
from tests import tagged_lookup_oracle as TL
from tests import zk_oracle as ZK
from tests.zk_oracle import add_zh_multiple, commit_coeffs, divide_linear, lincomb

R = O.R_MOD
N_BLINDERS = 21


class ZkLookupMixin(ZK.ZkMixin):
    def _zh_coeffs(self):
        """the Z_H multiple of every blinded polynomial, lowest coefficient first"""
        b = self.blinders
        return {"A": [b[1], b[0]], "B": [b[3], b[2]], "C": [b[5], b[4]], "Z": [b[8], b[7], b[6]],
                "F": [b[12], b[11]], "H1": [b[15], b[14], b[13]], "H2": [b[17], b[16]], "Z2": [b[20], b[19], b[18]]}

    def round_lookup(self):
        self._unblinded_round(super().round_lookup)  # sets Tl, F, H1, H2 from eta
        n, c = self.group_order, self._zh_coeffs()
        self.Fb, self.H1b, self.H2b = (add_zh_multiple(O.ifft(v), c[k], n)
                                       for k, v in (("F", self.F), ("H1", self.H1), ("H2", self.H2)))
        return tuple(commit_coeffs(self.setup, p) for p in (self.Fb, self.H1b, self.H2b))

    def round_2_lookup(self):
        self._unblinded_round(super().round_2_lookup)  # sets Z2 and checks that it closes
        self.Z2b = add_zh_multiple(O.ifft(self.Z2), self._zh_coeffs()["Z2"], self.group_order)
        return commit_coeffs(self.setup, self.Z2b)

    def round_3(self):
        n, pk, b = self.group_order, self.pk, self.blinders
        xs = [self.fft_cofactor * m % R for m in O.roots_of_unity(4 * n)]
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]
        zc = self._zh_coeffs()

        def blinded(values, name):
            """the blinded polynomial on the coset: values' extension + (c0 + c1 x + c2 x^2) Z_H(x)"""
            return [(e + ZK.poly_eval(zc[name], x) * zh) % R for e, x, zh in zip(self.fft_expand(values), xs, ZH_b)]

        A_b, B_b, C_b, Z_b = (blinded(v, k) for k, v in (("A", self.A), ("B", self.B), ("C", self.C), ("Z", self.Z)))
        F_b, H1_b, H2_b, Z2_b = (blinded(v, k) for k, v in (("F", self.F), ("H1", self.H1), ("H2", self.H2),
                                                             ("Z2", self.Z2)))
        T_b = self.fft_expand(self.Tl)
        sh = lambda v: v[4:] + v[:4]  # noqa: E731  (X -> wX on the 4x finer domain)
        Zw_b, Tw_b, H1w_b, Z2w_b = sh(Z_b), sh(T_b), sh(H1_b), sh(Z2_b)
        PI_b = self.fft_expand(self.PI)
        QL_b, QR_b, QM_b, QO_b, QC_b = (self.fft_expand(v) for v in (pk.QL, pk.QR, pk.QM, pk.QO, self._qc_tagged()))
        QC_k = [(e, self.fft_expand(col)) for e, col in pk.custom]
        S1_b, S2_b, S3_b = (self.fft_expand(v) for v in (pk.S1, pk.S2, pk.S3))
        QK_b = self.fft_expand(pk.qk)
        L0_b = self.fft_expand([1] + [0] * (n - 1))
        al, be, ga = self.alpha, self.beta, self.gamma
        eta, d, e = self.eta, self.delta, self.epsilon
        od, eod = (1 + d) % R, e * (1 + d) % R
        a2 = al * al % R
        a3, a4 = a2 * al % R, a2 * a2 % R
        a5 = a4 * al % R
        Q = []
        for j in range(4 * n):
            a, bb, c, x = A_b[j], B_b[j], C_b[j], xs[j]
            gate = (a * QL_b[j] + bb * QR_b[j] + a * bb % R * QM_b[j] + c * QO_b[j] + PI_b[j] + QC_b[j]
                    + sum(q[j] * CG.monomial(ex, a, bb, c) for ex, q in QC_k))
            p1 = (a + be * x + ga) * (bb + 2 * be * x + ga) % R * (c + 3 * be * x + ga) % R
            p2 = (a + be * S1_b[j] + ga) * (bb + be * S2_b[j] + ga) % R * (c + be * S3_b[j] + ga) % R
            lk1 = QK_b[j] * (a + eta * bb + eta * eta % R * c - F_b[j]) % R
            lk2 = (Z2_b[j] * od % R * (e + F_b[j]) % R * ((eod + T_b[j] + d * Tw_b[j]) % R)
                   - Z2w_b[j] * ((eod + H1_b[j] + d * H2_b[j]) % R) % R * ((eod + H2_b[j] + d * H1w_b[j]) % R)) % R
            lk3 = (Z2_b[j] - 1) * L0_b[j] % R
            num = (gate + al * (p1 * Z_b[j] - p2 * Zw_b[j]) + a2 * (Z_b[j] - 1) * L0_b[j]
                   + a3 * lk1 + a4 * lk2 + a5 * lk3) % R
            Q.append(num * O.inv0(ZH_b[j], R) % R)
        T = self.expanded_evals_to_coeffs(Q)
        assert T[3 * n + 6:] == [0] * (n - 6)  # deg T <= 3n + 5, as in plain zero-knowledge mode
        self.T = T
        b10, b11 = b[9], b[10]
        self.T1b = T[:n] + [b10]
        self.T2b = [(T[n] - b10) % R] + T[n + 1:2 * n] + [b11]
        self.T3b = [(T[2 * n] - b11) % R] + T[2 * n + 1:3 * n + 6]
        return tuple(commit_coeffs(self.setup, p) for p in (self.T1b, self.T2b, self.T3b))

    def round_4_lookup(self):
        fe, te, tw, h2e, h1w, z2w = super().round_4_lookup()  # the unblinded values, corrected here
        n, z, zc = self.group_order, self.zeta, self._zh_coeffs()
        zw = z * O.root_of_unity(n) % R
        zh = (pow(z, n, R) - 1) % R  # Z_H(zeta w) = Z_H(zeta)
        self.lk_ev = ((fe + ZK.poly_eval(zc["F"], z) * zh) % R, te, tw, (h2e + ZK.poly_eval(zc["H2"], z) * zh) % R,
                      (h1w + ZK.poly_eval(zc["H1"], zw) * zh) % R, (z2w + ZK.poly_eval(zc["Z2"], zw) * zh) % R)
        return self.lk_ev

    def round_5(self):
        n, pk = self.group_order, self.pk
        zeta, v = self.zeta, self.v
        al, be, ga = self.alpha, self.beta, self.gamma
        eta, d, e = self.eta, self.delta, self.epsilon
        a, b, c = self.a_eval, self.b_eval, self.c_eval
        s1, s2, zw = self.s1_eval, self.s2_eval, self.z_shifted_eval
        fe, te, tw, h2e, h1w, z2w = self.lk_ev
        od, eod = (1 + d) % R, e * (1 + d) % R
        zn = pow(zeta, n, R)
        ZH_ev = (zn - 1) % R
        L0_ev = ZH_ev * O.inv0(n * (zeta - 1), R) % R
        PI_ev = O.barycentric_eval(self.PI, zeta)
        c1 = (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al % R
        c2 = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
        a2 = al * al % R
        a3, a4 = a2 * al % R, a2 * a2 % R
        a5 = a4 * al % R
        al2l0 = a2 * L0_ev % R
        qc = self._qc_tagged()  # QC + alpha^3 eta^3 Q_T, and the custom terms at the evaluations
        for ex, col in pk.custom:
            m = CG.monomial(ex, a, b, c)
            qc = [(x + m * y) % R for x, y in zip(qc, col)]
        QL, QR, QM, QO, QC, S1, S2, S3, QK, Tc = (O.ifft(p) for p in (pk.QL, pk.QR, pk.QM, pk.QO, qc, pk.S1, pk.S2,
                                                                       pk.S3, pk.qk, self.Tl))
        hw = (eod + h2e + d * h1w) % R
        abc = (a + eta * b + eta * eta % R * c) % R
        v2, v3, v4, v5, v6, v7, v8 = (pow(v, k, R) for k in range(2, 9))
        # W_z numerator: ZkMixin's, with the lookup part of the linearisation
        #   a3 (abc - f) q_K + a4 (Z2' (1+d)(e+f)(e(1+d) + t + d t(zeta w)) - z2(zeta w)(e(1+d) + H1' + d h2) hw)
        #   + a5 L0(zeta) (Z2' - 1)
        # and v^6 (F' - f) + v^7 (T - t) + v^8 (H2' - h2)
        num = lincomb([(QL, a), (QR, b), (QM, a * b), (QO, c), (QC, 1), (self.Zb, c1 + al2l0), (S3, -c2 * be),
                       (self.T1b, -ZH_ev), (self.T2b, -ZH_ev * zn), (self.T3b, -ZH_ev * zn * zn),
                       (self.Ab, v), (self.Bb, v2), (self.Cb, v3), (S1, v4), (S2, v5),
                       (QK, a3 * (abc - fe)), (self.Z2b, a4 * od % R * (e + fe) % R * (eod + te + d * tw) + a5 * L0_ev),
                       (self.H1b, -a4 * z2w % R * hw), (self.Fb, v6), (Tc, v7), (self.H2b, v8)], n + 6)
        num[0] = (num[0] + PI_ev - c2 * (c + ga) - al2l0 - v * a - v2 * b - v3 * c - v4 * s1 - v5 * s2
                  - a4 * z2w % R * ((eod + d * h2e) % R) % R * hw - a5 * L0_ev - v6 * fe - v7 * te - v8 * h2e) % R
        Wz = divide_linear(num, zeta)
        numw = lincomb([(self.Zb, 1), (Tc, v), (self.H1b, v2), (self.Z2b, v3)], n + 3)
        numw[0] = (numw[0] - zw - v * tw - v2 * h1w - v3 * z2w) % R
        Wzw = divide_linear(numw, zeta * O.root_of_unity(n) % R)
        return commit_coeffs(self.setup, Wz), commit_coeffs(self.setup, Wzw)


class ZkLookupProver(ZkLookupMixin, TL.TaggedProver):
    def __init__(self, setup, pk, blinders, check: bool = True):
        super().__init__(setup, pk, check=check)
        assert len(blinders) == N_BLINDERS
        self.blinders = [int(x) % R for x in blinders]


def make_prover(setup, pk: TL.TaggedPreprocessed, blinders, check: bool = True) -> ZkLookupProver:
    return ZkLookupProver(setup, pk, blinders, check=check)


def prove(setup, pk: TL.TaggedPreprocessed, A, B, C, public_inputs, blinders, fast: bool = False) -> dict:
    """the oracle's zero-knowledge lookup proof (the dict of lookup_oracle); ``fast``: transforms by the C restatement
    (setup: an oracle.fast.Setup of at least n + 6 powers)"""
    if fast:
        with F.c_kernels():
            return make_prover(setup, pk, blinders).prove(A, B, C, public_inputs)
    return make_prover(setup, pk, blinders).prove(A, B, C, public_inputs)
