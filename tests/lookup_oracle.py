"""TEST INFRASTRUCTURE ONLY -- the oracle prover and trapdoor verifier with a lookup argument.

plookup (eprint 2020/315) in the cyclic, alternating-split form of PlonKup (eprint 2022/086), as DESIGN.md fixes it.
``LookupProver`` subclasses the custom-gate oracle prover (tests/custom_gate_oracle.py) and leaves the pinned oracle
untouched: it adds step 1L and Z2, and runs rounds 3-5 in the reference's style (``fft_expand``, the quotient on the 4n
coset, barycentric evaluations, the opening numerators on the coset).  s is built with ``sorted`` over table indices.
Running it inside ``oracle.fast.c_kernels()`` (``prove(..., fast=True)``) answers the transforms with the C
restatement."""
from __future__ import annotations

from dataclasses import dataclass, field

from oracle import fast as F
from oracle import plonk_oracle as O
from tests import custom_gate_oracle as CG

R = O.R_MOD
LOOKUP_FIELDS = ("f_1", "h1_1", "h2_1", "z2_1", "f_eval", "t_eval", "t_shifted_eval", "h2_eval", "h1_shifted_eval",
                 "z2_shifted_eval")


@dataclass
class LookupPreprocessed(CG.CustomPreprocessed):
    qk: list = field(default_factory=list)     # n values, 0 / 1
    table: list = field(default_factory=list)  # [t1, t2, t3], each padded to n by repeating the last row


def table_index(table) -> dict:
    """(t1, t2, t3) -> the lowest table index of that row"""
    idx = {}
    for j, row in enumerate(zip(*table)):
        idx.setdefault(row, j)
    return idx


class LookupProver(CG.CustomProver):
    def prove(self, A, B, C, public_inputs) -> dict:
        n = self.group_order
        tr = O.Transcript(b"plonk")
        self.PI = [(-int(v)) % R for v in public_inputs] + [0] * (n - len(public_inputs))
        a_1, b_1, c_1 = self.round_1(A, B, C)
        self.beta, self.gamma = tr.round_1(a_1, b_1, c_1)
        self.eta = tr.get_and_append_challenge(b"eta")
        f_1, h1_1, h2_1 = self.round_lookup()
        for lbl, p in ((b"f_1", f_1), (b"h1_1", h1_1), (b"h2_1", h2_1)):
            tr.append_point(lbl, p)
        self.delta, self.epsilon = tr.get_and_append_challenge(b"delta"), tr.get_and_append_challenge(b"epsilon")
        z_1 = self.round_2()
        z2_1 = self.round_2_lookup()
        tr.append_point(b"z_1", z_1)
        tr.append_point(b"z2_1", z2_1)
        self.alpha, self.fft_cofactor = tr.get_and_append_challenge(b"alpha"), tr.get_and_append_challenge(b"fft_cofactor")
        t_lo_1, t_mid_1, t_hi_1 = self.round_3()
        self.zeta = tr.round_3(t_lo_1, t_mid_1, t_hi_1)
        evals = self.round_4()
        lk_evals = self.round_4_lookup()
        for lbl, x in zip(O.PROOF_FIELDS[7:13] + LOOKUP_FIELDS[4:], tuple(evals) + lk_evals):
            tr.append_scalar(lbl.encode(), x)
        self.v = tr.get_and_append_challenge(b"v")
        W_z_1, W_zw_1 = self.round_5()
        vals = (a_1, b_1, c_1, z_1, t_lo_1, t_mid_1, t_hi_1) + tuple(evals) + (W_z_1, W_zw_1)
        out = dict(zip(O.PROOF_FIELDS, vals))
        out.update(zip(LOOKUP_FIELDS, (f_1, h1_1, h2_1, z2_1) + lk_evals))
        return out

    def round_1(self, A, B, C):
        out = super().round_1(A, B, C)
        idx = table_index(self.pk.table)
        self.J = []
        for i in range(self.group_order):
            if self.pk.qk[i]:
                row = (self.A[i], self.B[i], self.C[i])
                assert row in idx, "lookup row %d is not in the table" % i
                self.J.append(idx[row])
            else:
                self.J.append(0)
        return out

    def round_lookup(self):
        n, (t1, t2, t3), eta = self.group_order, self.pk.table, self.eta
        self.Tl = [(x + eta * y + eta * eta % R * z) % R for x, y, z in zip(t1, t2, t3)]
        self.F = [self.Tl[j] for j in self.J]
        s = [self.Tl[j] for j in sorted(list(range(n)) + self.J)]
        self.H1, self.H2 = s[0::2], s[1::2]
        return self.setup.commit(self.F), self.setup.commit(self.H1), self.setup.commit(self.H2)

    def round_2_lookup(self):
        n, d, e = self.group_order, self.delta, self.epsilon
        od, eod = (1 + d) % R, e * (1 + d) % R
        T, F_, H1, H2 = self.Tl, self.F, self.H1, self.H2
        Z2 = [1]
        for i in range(n):
            i1 = (i + 1) % n
            num = od * (e + F_[i]) % R * (eod + T[i] + d * T[i1]) % R
            den = (eod + H1[i] + d * H2[i]) % R * ((eod + H2[i] + d * H1[i1]) % R) % R
            Z2.append(Z2[-1] * num % R * O.inv0(den, R) % R)
        assert Z2.pop() == 1, "lookup grand product does not close"
        self.Z2 = Z2
        return self.setup.commit(Z2)

    def round_3(self):
        n, pk = self.group_order, self.pk
        k = self.fft_cofactor
        xs = [k * m % R for m in O.roots_of_unity(4 * n)]
        A_b, B_b, C_b = (self.fft_expand(v) for v in (self.A, self.B, self.C))
        PI_b = self.fft_expand(self.PI)
        QL_b, QR_b, QM_b, QO_b, QC_b = (self.fft_expand(v) for v in (pk.QL, pk.QR, pk.QM, pk.QO, pk.QC))
        QC_k = [(e, self.fft_expand(col)) for e, col in pk.custom]
        Z_b = self.fft_expand(self.Z)
        S1_b, S2_b, S3_b = (self.fft_expand(v) for v in (pk.S1, pk.S2, pk.S3))
        QK_b, T_b, F_b, H1_b, H2_b, Z2_b = (self.fft_expand(v) for v in (pk.qk, self.Tl, self.F, self.H1, self.H2, self.Z2))
        sh = lambda v: v[4:] + v[:4]  # noqa: E731  (X -> wX on the 4x finer domain)
        Zw_b, Tw_b, H1w_b, Z2w_b = sh(Z_b), sh(T_b), sh(H1_b), sh(Z2_b)
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]
        L0_b = self.fft_expand([1] + [0] * (n - 1))
        al, be, ga = self.alpha, self.beta, self.gamma
        eta, d, e = self.eta, self.delta, self.epsilon
        od, eod = (1 + d) % R, e * (1 + d) % R
        a2 = al * al % R
        a3, a4 = a2 * al % R, a2 * a2 % R
        a5 = a4 * al % R
        Q = []
        for j in range(4 * n):
            a, b, c, x = A_b[j], B_b[j], C_b[j], xs[j]
            gate = (a * QL_b[j] + b * QR_b[j] + a * b % R * QM_b[j] + c * QO_b[j] + PI_b[j] + QC_b[j]
                    + sum(q[j] * CG.monomial(ex, a, b, c) for ex, q in QC_k))
            p1 = (a + be * x + ga) * (b + 2 * be * x + ga) % R * (c + 3 * be * x + ga) % R
            p2 = (a + be * S1_b[j] + ga) * (b + be * S2_b[j] + ga) % R * (c + be * S3_b[j] + ga) % R
            lk1 = QK_b[j] * (a + eta * b + eta * eta % R * c - F_b[j]) % R
            lk2 = (Z2_b[j] * od % R * (e + F_b[j]) % R * ((eod + T_b[j] + d * Tw_b[j]) % R)
                   - Z2w_b[j] * ((eod + H1_b[j] + d * H2_b[j]) % R) % R * ((eod + H2_b[j] + d * H1w_b[j]) % R)) % R
            lk3 = (Z2_b[j] - 1) * L0_b[j] % R
            num = (gate + al * (p1 * Z_b[j] - p2 * Zw_b[j]) + a2 * (Z_b[j] - 1) * L0_b[j]
                   + a3 * lk1 + a4 * lk2 + a5 * lk3) % R
            Q.append(num * O.inv0(ZH_b[j], R) % R)
        T = self.expanded_evals_to_coeffs(Q)
        assert T[-n:] == [0] * n  # each lookup term has degree <= 3n: T still has three pieces
        self.T1c, self.T2c, self.T3c = T[:n], T[n:2 * n], T[2 * n:3 * n]
        self.T1, self.T2, self.T3 = O.fft(self.T1c), O.fft(self.T2c), O.fft(self.T3c)
        return self.setup.commit(self.T1), self.setup.commit(self.T2), self.setup.commit(self.T3)

    def round_4_lookup(self):
        z, w = self.zeta, O.root_of_unity(self.group_order)
        zw = z * w % R
        self.lk_ev = (O.barycentric_eval(self.F, z), O.barycentric_eval(self.Tl, z), O.barycentric_eval(self.Tl, zw),
                      O.barycentric_eval(self.H2, z), O.barycentric_eval(self.H1, zw), O.barycentric_eval(self.Z2, zw))
        return self.lk_ev

    def round_5(self):
        n, pk = self.group_order, self.pk
        zeta, v = self.zeta, self.v
        al, be, ga = self.alpha, self.beta, self.gamma
        eta, d, e = self.eta, self.delta, self.epsilon
        od, eod = (1 + d) % R, e * (1 + d) % R
        w = O.root_of_unity(n)
        xs = [self.fft_cofactor * m % R for m in O.roots_of_unity(4 * n)]
        L0_ev = (pow(zeta, n, R) - 1) * O.inv0(n * (zeta - 1), R) % R
        ZH_ev = (pow(zeta, n, R) - 1) % R
        T1_b, T2_b, T3_b = (self.fft_expand(t) for t in (self.T1, self.T2, self.T3))
        QL_b, QR_b, QM_b, QO_b, QC_b = (self.fft_expand(p) for p in (pk.QL, pk.QR, pk.QM, pk.QO, pk.QC))
        QC_k = [(ex, self.fft_expand(col)) for ex, col in pk.custom]
        Z_b, S1_b, S2_b, S3_b = (self.fft_expand(p) for p in (self.Z, pk.S1, pk.S2, pk.S3))
        A_b, B_b, C_b = (self.fft_expand(p) for p in (self.A, self.B, self.C))
        QK_b, T_b, F_b, H1_b, H2_b, Z2_b = (self.fft_expand(p) for p in (pk.qk, self.Tl, self.F, self.H1, self.H2, self.Z2))
        PI_ev = O.barycentric_eval(self.PI, zeta)
        a, b, c = self.a_eval, self.b_eval, self.c_eval
        s1, s2, zw = self.s1_eval, self.s2_eval, self.z_shifted_eval
        fe, te, tw, h2e, h1w, z2w = self.lk_ev
        c1 = (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al % R
        c2 = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
        m_k = [(CG.monomial(ex, a, b, c), q) for ex, q in QC_k]
        zn, z2n = pow(zeta, n, R), pow(zeta, 2 * n, R)
        a2 = al * al % R
        a3, a4 = a2 * al % R, a2 * a2 % R
        a5 = a4 * al % R
        hw = (eod + h2e + d * h1w) % R
        abc = (a + eta * b + eta * eta % R * c) % R
        v2, v3, v4, v5, v6, v7, v8 = (pow(v, k, R) for k in range(2, 9))
        Wz_b, Wzw_b, R_b = [], [], []
        for j in range(4 * n):
            r = (a * QL_b[j] + b * QR_b[j] + a * b % R * QM_b[j] + c * QO_b[j] + PI_ev + QC_b[j]
                 + sum(m * q[j] for m, q in m_k)
                 + c1 * Z_b[j] - c2 * ((c + be * S3_b[j] + ga) % R) + a2 * L0_ev % R * (Z_b[j] - 1)
                 - ZH_ev * ((T1_b[j] + zn * T2_b[j] + z2n * T3_b[j]) % R)
                 + a3 * QK_b[j] % R * (abc - fe)
                 + a4 * (Z2_b[j] * od % R * (e + fe) % R * ((eod + te + d * tw) % R)
                         - z2w * ((eod + H1_b[j] + d * h2e) % R) % R * hw)
                 + a5 * L0_ev % R * (Z2_b[j] - 1)) % R
            R_b.append(r)
            num = (r + v * (A_b[j] - a) + v2 * (B_b[j] - b) + v3 * (C_b[j] - c) + v4 * (S1_b[j] - s1)
                   + v5 * (S2_b[j] - s2) + v6 * (F_b[j] - fe) + v7 * (T_b[j] - te) + v8 * (H2_b[j] - h2e)) % R
            Wz_b.append(num * O.inv0(xs[j] - zeta, R) % R)
            numw = (Z_b[j] - zw + v * (T_b[j] - tw) + v2 * (H1_b[j] - h1w) + v3 * (Z2_b[j] - z2w)) % R
            Wzw_b.append(numw * O.inv0(xs[j] - zeta * w, R) % R)
        R_coeffs = self.expanded_evals_to_coeffs(R_b)
        assert R_coeffs[n:] == [0] * (3 * n)
        assert O.barycentric_eval(O.fft(R_coeffs[:n]), zeta) == 0
        Wz = self.expanded_evals_to_coeffs(Wz_b)
        assert Wz[n:] == [0] * (3 * n)
        Wzw = self.expanded_evals_to_coeffs(Wzw_b)
        assert Wzw[n:] == [0] * (3 * n)
        return self.setup.commit(O.fft(Wz[:n])), self.setup.commit(O.fft(Wzw[:n]))


def prove(setup, pk: LookupPreprocessed, A, B, C, public_inputs, fast: bool = False) -> dict:
    if fast:
        with F.c_kernels():
            return LookupProver(setup, pk).prove(A, B, C, public_inputs)
    return LookupProver(setup, pk).prove(A, B, C, public_inputs)


def proof_bytes(proof: dict) -> bytes:
    out = bytearray(O.proof_bytes(proof))
    for k in LOOKUP_FIELDS:
        v = proof[k]
        out += (int(v[0]).to_bytes(32, "big") + int(v[1]).to_bytes(32, "big")) if isinstance(v, tuple) \
            else int(v).to_bytes(32, "big")
    return bytes(out)


def proof_from_bytes(raw: bytes) -> dict:
    out = O.proof_from_bytes(raw[:768])
    w = [int.from_bytes(raw[i:i + 32], "big") for i in range(768, len(raw), 32)]
    vals = [(w[0], w[1]), (w[2], w[3]), (w[4], w[5]), (w[6], w[7])] + w[8:14]
    out.update(zip(LOOKUP_FIELDS, vals))
    return out


def challenges(proof: dict) -> dict:
    """the lookup transcript (plonkathon_b200/transcript.py LOOKUP_SCHEDULE), restated on the oracle's transcript"""
    tr = O.Transcript(b"plonk")
    steps = [(("a_1", "b_1", "c_1"), ("beta", "gamma", "eta")), (("f_1", "h1_1", "h2_1"), ("delta", "epsilon")),
             (("z_1", "z2_1"), ("alpha", "fft_cofactor")), (("t_lo_1", "t_mid_1", "t_hi_1"), ("zeta",)),
             (O.PROOF_FIELDS[7:13] + LOOKUP_FIELDS[4:], ("v",)), (("W_z_1", "W_zw_1"), ("u",))]
    out = {}
    for fields, drawn in steps:
        for f in fields:
            (tr.append_point if isinstance(proof[f], tuple) else tr.append_scalar)(f.encode(), proof[f])
        for lbl in drawn:
            out[lbl] = tr.get_and_append_challenge(lbl.encode())
    return out


def verify_proof_trapdoor(group_order: int, vk: dict, custom_pts, lookup_pts, proof: dict, public, tau: int) -> bool:
    """the batched verifier of a lookup proof with the final pairing equation checked through tau.
    lookup_pts: ([q_K], [t1], [t2], [t3]), None for the identity."""
    n = group_order
    ch = challenges(proof)
    be, ga, eta, d, e = ch["beta"], ch["gamma"], ch["eta"], ch["delta"], ch["epsilon"]
    al, zeta, v, u = ch["alpha"], ch["zeta"], ch["v"], ch["u"]
    w = O.root_of_unity(n)
    ZH = (pow(zeta, n, R) - 1) % R
    L0 = ZH * O.inv0(n * (zeta - 1), R) % R
    PI = sum((-p) * pow(w, i, R) % R * ZH % R * O.inv0(n * (zeta - pow(w, i, R)), R) for i, p in enumerate(public)) % R
    a, b, c = proof["a_eval"], proof["b_eval"], proof["c_eval"]
    s1, s2, zw = proof["s1_eval"], proof["s2_eval"], proof["z_shifted_eval"]
    fe, te, tw = proof["f_eval"], proof["t_eval"], proof["t_shifted_eval"]
    h2e, h1w, z2w = proof["h2_eval"], proof["h1_shifted_eval"], proof["z2_shifted_eval"]
    od, eod = (1 + d) % R, e * (1 + d) % R
    a2 = al * al % R
    a3, a4 = a2 * al % R, a2 * a2 % R
    a5 = a4 * al % R
    hw = (eod + h2e + d * h1w) % R
    v2, v3, v4, v5, v6, v7, v8 = (pow(v, k, R) for k in range(2, 9))
    sig = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
    r0 = (PI - L0 * a2 - sig * (c + ga) - a4 * z2w % R * ((eod + d * h2e) % R) % R * hw - a5 * L0) % R
    qk, t1, t2, t3 = lookup_pts
    pts = [
        (vk["Qm"], a * b), (vk["Ql"], a), (vk["Qr"], b), (vk["Qo"], c), (vk["Qc"], 1),
        *[(p, CG.monomial(ex, a, b, c)) for ex, p in custom_pts],
        (proof["z_1"], (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al
         + L0 * a2 + u),
        (vk["S3"], -sig * be),
        (proof["t_lo_1"], -ZH), (proof["t_mid_1"], -ZH * pow(zeta, n, R)), (proof["t_hi_1"], -ZH * pow(zeta, 2 * n, R)),
        (qk, a3 * ((a + eta * b + eta * eta % R * c - fe) % R)),
        (proof["z2_1"], a4 * od % R * (e + fe) % R * ((eod + te + d * tw) % R) + a5 * L0 + u * v3),
        (proof["h1_1"], -a4 * z2w % R * hw + u * v2),
        (t1, v7 + u * v), (t2, eta * (v7 + u * v)), (t3, eta * eta % R * (v7 + u * v)),
        (proof["a_1"], v), (proof["b_1"], v2), (proof["c_1"], v3), (vk["S1"], v4), (vk["S2"], v5),
        (proof["f_1"], v6), (proof["h2_1"], v8),
    ]
    Fp = O.ec_lincomb_naive([(p, k) for p, k in pts if p is not None])
    E = (-r0 + v * a + v2 * b + v3 * c + v4 * s1 + v5 * s2 + v6 * fe + v7 * te + v8 * h2e
         + u * (zw + v * tw + v2 * h1w + v3 * z2w)) % R
    lhs = O.g1_multiply(O.ec_lincomb_naive([(proof["W_z_1"], 1), (proof["W_zw_1"], u)]), tau)
    rhs = O.ec_lincomb_naive([(proof["W_z_1"], zeta), (proof["W_zw_1"], u * zeta % R * w), (Fp, 1),
                              (O.G1, -E % R)])
    return lhs == rhs


def preprocessed(c, S=None) -> LookupPreprocessed:
    """LookupPreprocessed of a plonkathon_b200.synthetic.ArrayCircuit with a lookup argument"""
    from plonkathon_b200 import synthetic as syn
    from plonkathon_b200.lookup import padded_table
    n = c.group_order
    S1, S2, S3 = S or syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    qk, table = c.lookup
    return LookupPreprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3, list(c.custom), list(qk),
                              padded_table([list(t) for t in table], n))
