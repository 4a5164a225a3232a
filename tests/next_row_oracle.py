"""TEST INFRASTRUCTURE ONLY -- the oracle prover and trapdoor verifier with custom gate terms over the next row.

A term (i, j, l, i', j', l') adds Q_k a^i b^j c^l a(wX)^i' b(wX)^j' c(wX)^l' to the gate constraint
(plonkathon_b200/custom_gates.py).  The reference has no such terms, so this extends tests/custom_gate_oracle.py in the
oracle's own structure: ``NextRowProver`` subclasses ``CustomProver`` and leaves it, and the pinned oracles, as they are.
  * round 1: the gate check reads row (i + 1) mod n;
  * round 3: the next-row wires on the 4n coset are A_b[4:] + A_b[:4] (B and C likewise), as Z(wX) is Zw_b;
  * round 4: A, B, C are also evaluated at zeta w, and the transcript absorbs them after z_shifted_eval;
  * round 5: with the wires fixed to their evaluations the terms are sum_k m_k Q_k(X), a constant selector folded into QC;
    the zeta w opening is (Z - z(zeta w)) + v (A - a(zeta w)) + v^2 (B - b(zeta w)) + v^3 (C - c(zeta w)).
Rounds 1-5 work on coefficient forms with the zero-knowledge blinders of zk_oracle.py (add_zh_multiple, divide_linear,
lincomb): with every blinder zero (``NextRowProver``) the commitments are those of the unblinded polynomials, and
``ZkNextRowProver`` takes 14 random ones, b12..b14 giving A, B, C a third blinder:
  A' = A + (b12 X^2 + b1 X + b2) Z_H,  B' = B + (b13 X^2 + b3 X + b4) Z_H,  C' = C + (b14 X^2 + b5 X + b6) Z_H,
  Z' = Z + (b7 X^2 + b8 X + b9) Z_H,  deg T <= 3n + 8,  T1' = T1 + b10 X^n, T2' = T2 - b10 + b11 X^n, T3' = T3 - b11.
The SRS needs n + 9 powers in zero-knowledge mode.  ``prove(..., fast=True)`` runs inside ``oracle.fast.c_kernels()``
with an ``oracle.fast.Setup``."""
from __future__ import annotations

from oracle import fast as F
from oracle import plonk_oracle as O
from tests import custom_gate_oracle as CG
from tests import zk_oracle as ZO

R = O.R_MOD
N_BLINDERS = 14
NEXT_ROW_FIELDS = ("a_shifted_eval", "b_shifted_eval", "c_shifted_eval")
ROUND4_FIELDS = O.PROOF_FIELDS[7:13] + NEXT_ROW_FIELDS


def padded(e):
    return tuple(e) + (0,) * (6 - len(e))


def monomial(exps, vals) -> int:
    """m_k over (a, b, c, a', b', c')"""
    m = 1
    for x, e in zip(vals, padded(exps)):
        m = m * pow(x, e, R) % R
    return m


def _commit(setup, coeffs):
    """[sum_i c_i tau^i] G, trailing zero coefficients left out (they need no SRS power)"""
    c = [int(x) % R for x in coeffs]
    while len(c) > 1 and c[-1] == 0:
        c.pop()
    return ZO.commit_coeffs(setup, c)


class NextRowProver(CG.CustomProver):
    """CustomProver with next-row terms in ``pk.custom`` (six exponents each, or three for a same-row term)"""

    def __init__(self, setup, pk, check: bool = True, blinders=None):
        super().__init__(setup, pk, check=check)
        self.blinders = [int(x) % R for x in blinders] if blinders is not None else [0] * N_BLINDERS
        assert len(self.blinders) == N_BLINDERS

    def prove(self, A, B, C, public_inputs) -> dict:
        """plonk_oracle.Prover.prove with round 4's three more evaluations in the transcript"""
        n = self.group_order
        tr = O.Transcript(b"plonk")
        self.PI = [(-int(v)) % R for v in public_inputs] + [0] * (n - len(public_inputs))
        a_1, b_1, c_1 = self.round_1(A, B, C)
        self.beta, self.gamma = tr.round_1(a_1, b_1, c_1)
        z_1 = self.round_2()
        self.alpha, self.fft_cofactor = tr.round_2(z_1)
        t_lo_1, t_mid_1, t_hi_1 = self.round_3()
        self.zeta = tr.round_3(t_lo_1, t_mid_1, t_hi_1)
        evals = self.round_4()
        for label, x in zip(ROUND4_FIELDS, evals):
            tr.append_scalar(label.encode(), x)
        self.v = tr.get_and_append_challenge(b"v")
        W_z_1, W_zw_1 = self.round_5()
        vals = (a_1, b_1, c_1, z_1, t_lo_1, t_mid_1, t_hi_1) + tuple(evals[:6]) + (W_z_1, W_zw_1)
        out = dict(zip(O.PROOF_FIELDS, vals))
        out.update(zip(NEXT_ROW_FIELDS, evals[6:]))
        return out

    def round_1(self, A, B, C):
        n, pk, b = self.group_order, self.pk, self.blinders
        A, B, C = ([int(v) % R for v in X] + [0] * (n - len(X)) for X in (A, B, C))
        if self.check:
            for i in range(n):
                i1 = (i + 1) % n
                vals = (A[i], B[i], C[i], A[i1], B[i1], C[i1])
                g = (A[i] * pk.QL[i] + B[i] * pk.QR[i] + A[i] * B[i] * pk.QM[i] + C[i] * pk.QO[i] + self.PI[i] + pk.QC[i]
                     + sum(col[i] * monomial(e, vals) for e, col in pk.custom))
                assert g % R == 0, "gate %d unsatisfied" % i
        self.A, self.B, self.C = A, B, C
        self.Ab, self.Bb, self.Cb = (ZO.add_zh_multiple(O.ifft(v), [b[2 * k + 1], b[2 * k], b[11 + k]], n)
                                     for k, v in enumerate((A, B, C)))
        return tuple(_commit(self.setup, p) for p in (self.Ab, self.Bb, self.Cb))

    def round_2(self):
        setup, self.setup = self.setup, ZO._NoCommit()
        try:
            O.Prover.round_2(self)  # sets self.Z and checks Z_n == 1
        finally:
            self.setup = setup
        b = self.blinders
        self.Zb = ZO.add_zh_multiple(O.ifft(self.Z), [b[8], b[7], b[6]], self.group_order)
        return _commit(self.setup, self.Zb)

    def round_3(self):
        n, pk, b = self.group_order, self.pk, self.blinders
        k = self.fft_cofactor
        xs = [k * m % R for m in O.roots_of_unity(4 * n)]
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]

        def blinded(vals, c2, c1, c0):  # the coset values of vals + (c2 X^2 + c1 X + c0) Z_H
            return [(e + ((c2 * x + c1) * x + c0) * zh) % R for e, x, zh in zip(self.fft_expand(vals), xs, ZH_b)]
        A_b, B_b, C_b = (blinded(v, b[11 + w], b[2 * w], b[2 * w + 1]) for w, v in enumerate((self.A, self.B, self.C)))
        Z_b = blinded(self.Z, b[6], b[7], b[8])
        sh = lambda v: v[4:] + v[:4]  # noqa: E731  (X -> wX on the 4x finer domain)
        Aw_b, Bw_b, Cw_b, Zw_b = sh(A_b), sh(B_b), sh(C_b), sh(Z_b)
        PI_b = self.fft_expand(self.PI)
        QL_b, QR_b, QM_b, QO_b, QC_b = (self.fft_expand(v) for v in (pk.QL, pk.QR, pk.QM, pk.QO, pk.QC))
        QK_b = [(e, self.fft_expand(col)) for e, col in pk.custom]
        S1_b, S2_b, S3_b = (self.fft_expand(v) for v in (pk.S1, pk.S2, pk.S3))
        L0_b = self.fft_expand([1] + [0] * (n - 1))
        al, be, ga = self.alpha, self.beta, self.gamma
        Q = []
        for j in range(4 * n):
            a, bb, c, x = A_b[j], B_b[j], C_b[j], xs[j]
            vals = (a, bb, c, Aw_b[j], Bw_b[j], Cw_b[j])
            gate = (a * QL_b[j] + bb * QR_b[j] + a * bb % R * QM_b[j] + c * QO_b[j] + PI_b[j] + QC_b[j]
                    + sum(q[j] * monomial(e, vals) for e, q in QK_b))
            p1 = (a + be * x + ga) * (bb + 2 * be * x + ga) % R * (c + 3 * be * x + ga) % R
            p2 = (a + be * S1_b[j] + ga) * (bb + be * S2_b[j] + ga) % R * (c + be * S3_b[j] + ga) % R
            num = (gate + al * (p1 * Z_b[j] - p2 * Zw_b[j]) + al * al % R * (Z_b[j] - 1) * L0_b[j]) % R
            Q.append(num * O.inv0(ZH_b[j], R) % R)
        T = self.expanded_evals_to_coeffs(Q)
        assert T[3 * n + 9:] == [0] * (n - 9)  # deg T <= 3n + 8
        if not any(b):
            assert T[3 * n:] == [0] * n  # without blinders: three pieces of n coefficients
        b10, b11 = b[9], b[10]
        self.T1b = T[:n] + [b10]
        self.T2b = [(T[n] - b10) % R] + T[n + 1:2 * n] + [b11]
        self.T3b = [(T[2 * n] - b11) % R] + T[2 * n + 1:3 * n + 9]
        return tuple(_commit(self.setup, p) for p in (self.T1b, self.T2b, self.T3b))

    def round_4(self):
        """the blinded wires at zeta, S1, S2 at zeta, and Z, A, B, C at zeta w (barycentric for S1, S2, Horner for the
        coefficient forms)"""
        n, z = self.group_order, self.zeta
        zw = z * O.root_of_unity(n) % R
        self.a_eval, self.b_eval, self.c_eval = (ZO.poly_eval(p, z) for p in (self.Ab, self.Bb, self.Cb))
        self.s1_eval = O.barycentric_eval(self.pk.S1, z)
        self.s2_eval = O.barycentric_eval(self.pk.S2, z)
        self.z_shifted_eval = ZO.poly_eval(self.Zb, zw)
        self.shifted = tuple(ZO.poly_eval(p, zw) for p in (self.Ab, self.Bb, self.Cb))
        return (self.a_eval, self.b_eval, self.c_eval, self.s1_eval, self.s2_eval, self.z_shifted_eval) + self.shifted

    def round_5(self):
        n, pk = self.group_order, self.pk
        zeta, v = self.zeta, self.v
        al, be, ga = self.alpha, self.beta, self.gamma
        a, b, c = self.a_eval, self.b_eval, self.c_eval
        s1, s2, zw = self.s1_eval, self.s2_eval, self.z_shifted_eval
        aw, bw, cw = self.shifted
        zn = pow(zeta, n, R)
        ZH_ev = (zn - 1) % R
        L0_ev = ZH_ev * O.inv0(n * (zeta - 1), R) % R
        PI_ev = O.barycentric_eval(self.PI, zeta)
        c1 = (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al % R
        c2 = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
        al2l0 = al * al % R * L0_ev % R
        qc = list(pk.QC)
        for e, col in pk.custom:  # the terms at the evaluations: a constant selector, like QC
            m = monomial(e, (a, b, c, aw, bw, cw))
            qc = [(x + m * y) % R for x, y in zip(qc, col)]
        QL, QR, QM, QO, QC, S1, S2, S3 = (O.ifft(p) for p in (pk.QL, pk.QR, pk.QM, pk.QO, qc, pk.S1, pk.S2, pk.S3))
        v2, v3, v4, v5 = (pow(v, e, R) for e in (2, 3, 4, 5))
        num = ZO.lincomb([(QL, a), (QR, b), (QM, a * b), (QO, c), (QC, 1), (self.Zb, c1 + al2l0), (S3, -c2 * be),
                          (self.T1b, -ZH_ev), (self.T2b, -ZH_ev * zn), (self.T3b, -ZH_ev * zn * zn),
                          (self.Ab, v), (self.Bb, v2), (self.Cb, v3), (S1, v4), (S2, v5)], n + 9)
        num[0] = (num[0] + PI_ev - c2 * (c + ga) - al2l0 - v * a - v2 * b - v3 * c - v4 * s1 - v5 * s2) % R
        Wz = ZO.divide_linear(num, zeta)
        numw = ZO.lincomb([(self.Zb, 1), (self.Ab, v), (self.Bb, v2), (self.Cb, v3)], n + 3)
        numw[0] = (numw[0] - zw - v * aw - v2 * bw - v3 * cw) % R
        Wzw = ZO.divide_linear(numw, zeta * O.root_of_unity(n) % R)
        return _commit(self.setup, Wz), _commit(self.setup, Wzw)


class ZkNextRowProver(NextRowProver):
    """zero-knowledge mode of a next-row circuit: the 14 blinders b1..b14 (zk_oracle.py's 11, then b12..b14)"""

    def __init__(self, setup, pk, blinders, check: bool = True):
        assert len(blinders) == N_BLINDERS
        super().__init__(setup, pk, check=check, blinders=blinders)


def prove(setup, pk, A, B, C, public_inputs, blinders=None, fast: bool = False, check: bool = True) -> dict:
    """the oracle's proof of a next-row circuit (``blinders``: 14 for zero-knowledge mode); ``fast``: transforms by the C
    restatement (setup: an oracle.fast.Setup, of n + 9 powers with blinders)"""
    cls = NextRowProver if blinders is None else ZkNextRowProver
    if fast:
        with F.c_kernels():
            return cls(setup, pk, blinders=blinders, check=check).prove(A, B, C, public_inputs)
    return cls(setup, pk, blinders=blinders, check=check).prove(A, B, C, public_inputs)


def proof_bytes(proof: dict) -> bytes:
    return O.proof_bytes(proof) + b"".join(int(proof[k]).to_bytes(32, "big") for k in NEXT_ROW_FIELDS)


def proof_from_bytes(raw: bytes) -> dict:
    out = O.proof_from_bytes(raw[:768])
    out.update(zip(NEXT_ROW_FIELDS, [int.from_bytes(raw[i:i + 32], "big") for i in range(768, 864, 32)]))
    return out


def challenges(proof: dict) -> dict:
    """the next-row transcript (plonkathon_b200/transcript.py NEXT_ROW_SCHEDULE), restated on the oracle's transcript"""
    tr = O.Transcript(b"plonk")
    steps = [(("a_1", "b_1", "c_1"), ("beta", "gamma")), (("z_1",), ("alpha", "fft_cofactor")),
             (("t_lo_1", "t_mid_1", "t_hi_1"), ("zeta",)), (ROUND4_FIELDS, ("v",)), (("W_z_1", "W_zw_1"), ("u",))]
    out = {}
    for fields, drawn in steps:
        for f in fields:
            (tr.append_point if isinstance(proof[f], tuple) else tr.append_scalar)(f.encode(), proof[f])
        for lbl in drawn:
            out[lbl] = tr.get_and_append_challenge(lbl.encode())
    return out


def verify_proof_trapdoor(group_order: int, vk: dict, custom_pts, proof: dict, public, tau: int) -> bool:
    """the batched verifier of a next-row proof with the final pairing equation checked through tau.  custom_pts:
    (exponents, [Q_k]) in the prover's order"""
    n = group_order
    ch = challenges(proof)
    be, ga, al, zeta, v, u = ch["beta"], ch["gamma"], ch["alpha"], ch["zeta"], ch["v"], ch["u"]
    w = O.root_of_unity(n)
    ZH = (pow(zeta, n, R) - 1) % R
    L0 = ZH * O.inv0(n * (zeta - 1), R) % R
    PI = sum((-p) * pow(w, i, R) % R * ZH % R * O.inv0(n * (zeta - pow(w, i, R)), R) for i, p in enumerate(public)) % R
    a, b, c = proof["a_eval"], proof["b_eval"], proof["c_eval"]
    s1, s2, zw = proof["s1_eval"], proof["s2_eval"], proof["z_shifted_eval"]
    aw, bw, cw = (proof[k] for k in NEXT_ROW_FIELDS)
    a2 = al * al % R
    v2, v3, v4, v5 = (pow(v, k, R) for k in range(2, 6))
    sig = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
    r0 = (PI - L0 * a2 - sig * (c + ga)) % R
    pts = [
        (vk["Qm"], a * b), (vk["Ql"], a), (vk["Qr"], b), (vk["Qo"], c), (vk["Qc"], 1),
        *[(p, monomial(e, (a, b, c, aw, bw, cw))) for e, p in custom_pts],
        (proof["z_1"], (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al
         + L0 * a2 + u),
        (vk["S3"], -sig * be),
        (proof["t_lo_1"], -ZH), (proof["t_mid_1"], -ZH * pow(zeta, n, R)), (proof["t_hi_1"], -ZH * pow(zeta, 2 * n, R)),
        (proof["a_1"], v + u * v), (proof["b_1"], v2 + u * v2), (proof["c_1"], v3 + u * v3),
        (vk["S1"], v4), (vk["S2"], v5),
    ]
    Fp = O.ec_lincomb_naive([(p, k % R) for p, k in pts if p is not None])
    E = (-r0 + v * a + v2 * b + v3 * c + v4 * s1 + v5 * s2 + u * (zw + v * aw + v2 * bw + v3 * cw)) % R
    lhs = O.g1_multiply(O.ec_lincomb_naive([(proof["W_z_1"], 1), (proof["W_zw_1"], u)]), tau)
    rhs = O.ec_lincomb_naive([(proof["W_z_1"], zeta), (proof["W_zw_1"], u * zeta % R * w), (Fp, 1), (O.G1, -E % R)])
    return lhs == rhs


def preprocessed(c, S=None) -> CG.CustomPreprocessed:
    """CustomPreprocessed of a plonkathon_b200.synthetic.ArrayCircuit with next-row terms"""
    return CG.preprocessed(c, S)
