"""TEST INFRASTRUCTURE ONLY -- the oracle prover in zero-knowledge mode, with explicit blinders.

The blinding of the PLONK paper (eprint 2019/953, prover rounds 1-3), b1..b11 = blinders[0..10], Z_H = X^n - 1:
  A' = A + (b1 X + b2) Z_H,  B' = B + (b3 X + b4) Z_H,  C' = C + (b5 X + b6) Z_H,  Z' = Z + (b7 X^2 + b8 X + b9) Z_H,
  T = (gate + alpha perm + alpha^2 L0 (Z' - 1)) / Z_H  (degree <= 3n + 5), cut at n and 2n, then
  T1' = T1 + b10 X^n,  T2' = T2 - b10 + b11 X^n,  T3' = T3 - b11.
The reference has no blinding, so this extends oracle/plonk_oracle.py without following a reference file.  ``ZkMixin``
goes in front of ``plonk_oracle.Prover`` (``ZkProver``) or ``custom_gate_oracle.CustomProver`` (``ZkCustomProver``), which
stay as they are: rounds 1-2 run the parent's rounds (witness checks, grand product) and commit the blinded polynomials in
monomial form instead; round 3 adds the Z_H multiples on the coset; round 4 corrects the parent's evaluations; round 5
builds the linearisation and the two openings in coefficient form (the blinded polynomials have more than n
coefficients, so the parent's n-point Lagrange round 5 does not apply).  The SRS needs n + 6 powers.  ``prove(...,
fast=True)`` runs inside ``oracle.fast.c_kernels()`` with an ``oracle.fast.Setup``, whose transforms and MSMs are the C
restatement."""
from __future__ import annotations

from oracle import c_oracle as CO
from oracle import fast as F
from oracle import plonk_oracle as O
from tests import custom_gate_oracle as CG

R = O.R_MOD
N_BLINDERS = 11


def commit_coeffs(setup, coeffs):
    """[sum_i c_i tau^i] G: plonk_oracle.Setup.commit_coeffs, or the C lincomb over an oracle.fast.Setup's points"""
    coeffs = [int(c) % R for c in coeffs]
    if isinstance(setup, F.Setup):
        if len(coeffs) > setup.pts.shape[0]:
            raise Exception("Not enough powers in setup")
        return CO.g1_lincomb(setup.pts[:len(coeffs)], F._to_np(coeffs))
    if len(coeffs) > len(setup.powers_of_x):
        raise Exception("Not enough powers in setup")
    return setup.commit_coeffs(coeffs)


def add_zh_multiple(coeffs, c, n):
    """coeffs (zero padded to n + len(c)) + (c[0] + c[1] X + ...) (X^n - 1)"""
    out = [int(x) % R for x in coeffs] + [0] * (n + len(c) - len(coeffs))
    for i, ci in enumerate(c):
        out[i] = (out[i] - ci) % R
        out[n + i] = (out[n + i] + ci) % R
    return out


def poly_eval(coeffs, x):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % R
    return acc


def divide_linear(num, point):
    """num / (X - point) by synthetic division; asserts the remainder is zero"""
    q = [0] * (len(num) - 1)
    acc = 0
    for i in range(len(num) - 1, 0, -1):
        acc = (acc * point + num[i]) % R
        q[i - 1] = acc
    assert (acc * point + num[0]) % R == 0, "opening numerator is not divisible by (X - point)"
    return q


def lincomb(terms, length):
    out = [0] * length
    for vec, w in terms:
        w %= R
        if w:
            for i, x in enumerate(vec):
                out[i] = (out[i] + w * x) % R
    return out


class _NoCommit:
    """stands in for the setup while the parent's round 1 / 2 runs: its Lagrange commitments of the unblinded
    polynomials are not part of a zero-knowledge proof"""

    def commit(self, values):
        return None


class ZkMixin:
    blinders: list

    def _unblinded_round(self, fn, *args):
        setup, self.setup = self.setup, _NoCommit()
        try:
            fn(*args)
        finally:
            self.setup = setup

    def round_1(self, A, B, C):
        self._unblinded_round(super().round_1, A, B, C)  # sets self.A/B/C and checks the gates
        n, b = self.group_order, self.blinders
        self.Ab, self.Bb, self.Cb = (add_zh_multiple(O.ifft(v), [b[2 * k + 1], b[2 * k]], n)
                                     for k, v in enumerate((self.A, self.B, self.C)))
        return tuple(commit_coeffs(self.setup, p) for p in (self.Ab, self.Bb, self.Cb))

    def round_2(self):
        self._unblinded_round(super().round_2)  # sets self.Z and checks Z_n == 1
        b = self.blinders
        self.Zb = add_zh_multiple(O.ifft(self.Z), [b[8], b[7], b[6]], self.group_order)
        return commit_coeffs(self.setup, self.Zb)

    def round_3(self):
        n, pk, b = self.group_order, self.pk, self.blinders
        k = self.fft_cofactor
        xs = [k * m % R for m in O.roots_of_unity(4 * n)]
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]
        A_b, B_b, C_b = ([(e + (b[2 * w] * x + b[2 * w + 1]) * zh) % R for e, x, zh in zip(self.fft_expand(v), xs, ZH_b)]
                         for w, v in enumerate((self.A, self.B, self.C)))
        Z_b = [(e + ((b[6] * x + b[7]) * x + b[8]) * zh) % R for e, x, zh in zip(self.fft_expand(self.Z), xs, ZH_b)]
        Zw_b = Z_b[4:] + Z_b[:4]  # Z'(wX): the blinded values on the coset shifted by w
        PI_b = self.fft_expand(self.PI)
        QL_b, QR_b, QM_b, QO_b, QC_b = (self.fft_expand(v) for v in (pk.QL, pk.QR, pk.QM, pk.QO, pk.QC))
        QK_b = [(e, self.fft_expand(col)) for e, col in getattr(pk, "custom", ())]
        S1_b, S2_b, S3_b = (self.fft_expand(v) for v in (pk.S1, pk.S2, pk.S3))
        L0_b = self.fft_expand([1] + [0] * (n - 1))
        al, be, ga = self.alpha, self.beta, self.gamma
        Q = []
        for j in range(4 * n):
            a, bb, c, x = A_b[j], B_b[j], C_b[j], xs[j]
            gate = (a * QL_b[j] + bb * QR_b[j] + a * bb % R * QM_b[j] + c * QO_b[j] + PI_b[j] + QC_b[j]
                    + sum(q[j] * CG.monomial(e, a, bb, c) for e, q in QK_b))
            p1 = (a + be * x + ga) * (bb + 2 * be * x + ga) % R * (c + 3 * be * x + ga) % R
            p2 = (a + be * S1_b[j] + ga) * (bb + be * S2_b[j] + ga) % R * (c + be * S3_b[j] + ga) % R
            num = (gate + al * (p1 * Z_b[j] - p2 * Zw_b[j]) + al * al % R * (Z_b[j] - 1) * L0_b[j]) % R
            Q.append(num * O.inv0(ZH_b[j], R) % R)
        T = self.expanded_evals_to_coeffs(Q)
        assert T[3 * n + 6:] == [0] * (n - 6)  # deg T <= 3n + 5
        self.T = T
        b10, b11 = b[9], b[10]
        self.T1b = T[:n] + [b10]
        self.T2b = [(T[n] - b10) % R] + T[n + 1:2 * n] + [b11]
        self.T3b = [(T[2 * n] - b11) % R] + T[2 * n + 1:3 * n + 6]
        return tuple(commit_coeffs(self.setup, p) for p in (self.T1b, self.T2b, self.T3b))

    def round_4(self):
        super().round_4()  # the unblinded evaluations, corrected below
        n, z, b = self.group_order, self.zeta, self.blinders
        zw = z * O.root_of_unity(n) % R
        zh = (pow(z, n, R) - 1) % R
        self.a_eval = (self.a_eval + (b[0] * z + b[1]) * zh) % R
        self.b_eval = (self.b_eval + (b[2] * z + b[3]) * zh) % R
        self.c_eval = (self.c_eval + (b[4] * z + b[5]) * zh) % R
        self.z_shifted_eval = (self.z_shifted_eval + ((b[6] * zw + b[7]) * zw + b[8]) * zh) % R
        return (self.a_eval, self.b_eval, self.c_eval, self.s1_eval, self.s2_eval, self.z_shifted_eval)

    def round_5(self):
        n, pk = self.group_order, self.pk
        zeta, v = self.zeta, self.v
        al, be, ga = self.alpha, self.beta, self.gamma
        a, b, c = self.a_eval, self.b_eval, self.c_eval
        s1, s2, zw = self.s1_eval, self.s2_eval, self.z_shifted_eval
        zn = pow(zeta, n, R)
        ZH_ev = (zn - 1) % R
        L0_ev = ZH_ev * O.inv0(n * (zeta - 1), R) % R
        PI_ev = O.barycentric_eval(self.PI, zeta)
        c1 = (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al % R
        c2 = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
        al2l0 = al * al % R * L0_ev % R
        qc = list(pk.QC)
        for e, col in getattr(pk, "custom", ()):  # custom terms at the evaluations: a constant selector, like QC
            m = CG.monomial(e, a, b, c)
            qc = [(x + m * y) % R for x, y in zip(qc, col)]
        QL, QR, QM, QO, QC, S1, S2, S3 = (O.ifft(p) for p in (pk.QL, pk.QR, pk.QM, pk.QO, qc, pk.S1, pk.S2, pk.S3))
        v2, v3, v4, v5 = (pow(v, e, R) for e in (2, 3, 4, 5))
        # W_z numerator = R + v (A' - a) + v^2 (B' - b) + v^3 (C' - c) + v^4 (S1 - s1) + v^5 (S2 - s2), with
        # R = a QL + b QR + ab QM + c QO + QC + PI(zeta) + c1 Z' - c2 (c + beta S3 + gamma) + alpha^2 L0(zeta) (Z' - 1)
        #     - Z_H(zeta) (T1' + zeta^n T2' + zeta^2n T3')
        num = lincomb([(QL, a), (QR, b), (QM, a * b), (QO, c), (QC, 1), (self.Zb, c1 + al2l0), (S3, -c2 * be),
                       (self.T1b, -ZH_ev), (self.T2b, -ZH_ev * zn), (self.T3b, -ZH_ev * zn * zn),
                       (self.Ab, v), (self.Bb, v2), (self.Cb, v3), (S1, v4), (S2, v5)], n + 6)
        num[0] = (num[0] + PI_ev - c2 * (c + ga) - al2l0 - v * a - v2 * b - v3 * c - v4 * s1 - v5 * s2) % R
        Wz = divide_linear(num, zeta)
        Wzw = divide_linear([(self.Zb[0] - zw) % R] + self.Zb[1:], zeta * O.root_of_unity(n) % R)
        return commit_coeffs(self.setup, Wz), commit_coeffs(self.setup, Wzw)


class ZkProver(ZkMixin, O.Prover):
    def __init__(self, setup, pk, blinders, check: bool = True):
        super().__init__(setup, pk, check=check)
        assert len(blinders) == N_BLINDERS
        self.blinders = [int(x) % R for x in blinders]


class ZkCustomProver(ZkMixin, CG.CustomProver):
    def __init__(self, setup, pk, blinders, check: bool = True):
        super().__init__(setup, pk, check=check)
        assert len(blinders) == N_BLINDERS
        self.blinders = [int(x) % R for x in blinders]


def make_prover(setup, pk, blinders, check: bool = True):
    cls = ZkCustomProver if isinstance(pk, CG.CustomPreprocessed) else ZkProver
    return cls(setup, pk, blinders, check=check)


def prove(setup, pk, A, B, C, public_inputs, blinders, fast: bool = False, check: bool = True) -> dict:
    """the oracle's zero-knowledge proof; ``fast``: transforms by the C restatement (setup: an oracle.fast.Setup of at
    least n + 6 powers)"""
    if fast:
        with F.c_kernels():
            return make_prover(setup, pk, blinders, check).prove(A, B, C, public_inputs)
    return make_prover(setup, pk, blinders, check).prove(A, B, C, public_inputs)
