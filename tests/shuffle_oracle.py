"""TEST INFRASTRUCTURE ONLY -- the oracle prover and trapdoor verifier with a shuffle.

Two boolean selectors q_in, q_out claim that {(a_i, b_i, c_i) : q_in[i] = 1} and {(a_i, b_i, c_i) : q_out[i] = 1} are
equal multisets (plonkathon_b200/shuffle.py).  The reference has no shuffle, so this extends tests/next_row_oracle.py in
the oracle's own structure: ``ShuffleProver`` subclasses ``NextRowProver`` with every blinder zero, which proves a circuit
with same-row terms, next-row terms or none, and leaves it, the custom-gate oracle and the pinned oracles as they are.
  * round 1: the two multisets are compared exactly (sorted tuples) before anything is proved;
  * after beta, gamma the transcript draws theta, kappa; with w_i = a_i + theta b_i + theta^2 c_i,
    Z3_0 = 1, Z3_(i+1) = Z3_i (1 + q_in[i](kappa + w_i - 1)) / (1 + q_out[i](kappa + w_i - 1)), and Z3_n == 1;
  * round 3: alpha^3 [Z3(wX)(1 + Q_out(K + W - 1)) - Z3(1 + Q_in(K + W - 1))] + alpha^4 L0 (Z3 - 1) joins the quotient's
    evaluations on the 4n coset before they go back to coefficients;
  * round 4: Q_in at zeta and Z3 at zeta w, absorbed last;
  * round 5: [Q_out] and [Z3] in the linearisation, Q_in opened at zeta (v^6), Z3 at zeta w (v, or v^4 after A, B, C
    on a next-row circuit).
``prove(..., fast=True)`` runs inside ``oracle.fast.c_kernels()`` with an ``oracle.fast.Setup``."""
from __future__ import annotations

from dataclasses import dataclass, field

from oracle import fast as F
from oracle import plonk_oracle as O
from tests import custom_gate_oracle as CG
from tests import next_row_oracle as NR
from tests import zk_oracle as ZO

R = O.R_MOD
SHUFFLE_FIELDS = ("z3_1", "qin_eval", "z3_shifted_eval")
NOT_A_SHUFFLE = "shuffle: the q_in rows and the q_out rows are not permutations of each other"


@dataclass
class ShufflePreprocessed(CG.CustomPreprocessed):
    q_in: list = field(default_factory=list)   # n values, 0 or 1
    q_out: list = field(default_factory=list)


def is_next_row(pk) -> bool:
    return any(any(NR.padded(e)[3:]) for e, _ in pk.custom)


def round4_fields(next_row: bool):
    return O.PROOF_FIELDS[7:13] + (NR.NEXT_ROW_FIELDS if next_row else ()) + SHUFFLE_FIELDS[1:]


class ShuffleProver(NR.NextRowProver):
    """NextRowProver (no blinders) with the shuffle of ``pk.q_in``, ``pk.q_out``"""

    def __init__(self, setup, pk: ShufflePreprocessed, check: bool = True):
        super().__init__(setup, pk, check=check)
        self.next_row = is_next_row(pk)
        self._extra = None

    def prove(self, A, B, C, public_inputs) -> dict:
        n = self.group_order
        tr = O.Transcript(b"plonk")
        self.PI = [(-int(v)) % R for v in public_inputs] + [0] * (n - len(public_inputs))
        a_1, b_1, c_1 = self.round_1(A, B, C)
        self.beta, self.gamma = tr.round_1(a_1, b_1, c_1)
        self.theta = tr.get_and_append_challenge(b"theta")
        self.kappa = tr.get_and_append_challenge(b"kappa")
        z_1, z3_1 = self.round_2()
        tr.append_point(b"z_1", z_1)
        tr.append_point(b"z3_1", z3_1)
        self.alpha = tr.get_and_append_challenge(b"alpha")
        self.fft_cofactor = tr.get_and_append_challenge(b"fft_cofactor")
        t_lo_1, t_mid_1, t_hi_1 = self.round_3()
        self.zeta = tr.round_3(t_lo_1, t_mid_1, t_hi_1)
        evals = self.round_4()
        labels = round4_fields(self.next_row)
        for label, x in zip(labels, evals):
            tr.append_scalar(label.encode(), x)
        self.v = tr.get_and_append_challenge(b"v")
        W_z_1, W_zw_1 = self.round_5()
        vals = (a_1, b_1, c_1, z_1, t_lo_1, t_mid_1, t_hi_1) + tuple(evals[:6]) + (W_z_1, W_zw_1)
        out = dict(zip(O.PROOF_FIELDS, vals))
        out.update(zip(labels[6:], evals[6:]))
        out["z3_1"] = z3_1
        return out

    def round_1(self, A, B, C):
        n, pk = self.group_order, self.pk
        cols = [[int(v) % R for v in X] + [0] * (n - len(X)) for X in (A, B, C)]
        side = lambda q: sorted(tuple(c[i] for c in cols) for i in range(n) if q[i])  # noqa: E731
        assert side(pk.q_in) == side(pk.q_out), NOT_A_SHUFFLE
        return super().round_1(A, B, C)

    def _w(self, i):
        th = self.theta
        return (self.A[i] + th * self.B[i] + th * th % R * self.C[i]) % R

    def round_2(self):
        z_1 = super().round_2()
        n, pk = self.group_order, self.pk
        Z3 = [1]
        for i in range(n):
            t = (self.kappa + self._w(i)) % R
            num = t if pk.q_in[i] else 1
            den = t if pk.q_out[i] else 1
            Z3.append(Z3[-1] * num % R * O.inv0(den, R) % R)
        assert Z3.pop() == 1, NOT_A_SHUFFLE
        self.Z3 = Z3
        self.Z3c = O.ifft(Z3)
        return z_1, NR._commit(self.setup, self.Z3c)

    def expanded_evals_to_coeffs(self, x):
        """the quotient's evaluations gain the shuffle terms (self._extra) on their way back to coefficients"""
        if self._extra is not None:
            x = [(a + b) % R for a, b in zip(x, self._extra)]
        return super().expanded_evals_to_coeffs(x)

    def round_3(self):
        n, pk = self.group_order, self.pk
        k = self.fft_cofactor
        xs = [k * m % R for m in O.roots_of_unity(4 * n)]
        ZH_b = [(pow(x, n, R) - 1) % R for x in xs]
        A_b, B_b, C_b = (self.fft_expand(v) for v in (self.A, self.B, self.C))
        QI_b, QO_b = self.fft_expand(pk.q_in), self.fft_expand(pk.q_out)
        Z3_b = self.fft_expand(self.Z3)
        Z3w_b = Z3_b[4:] + Z3_b[:4]
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
            return super().round_3()
        finally:
            self._extra = None

    def round_4(self):
        evals = super().round_4()  # the six plain evaluations, then A, B, C at zeta w
        zw = self.zeta * O.root_of_unity(self.group_order) % R
        self.qin_eval = O.barycentric_eval(self.pk.q_in, self.zeta)
        self.z3_shifted_eval = ZO.poly_eval(self.Z3c, zw)
        return tuple(evals[:9] if self.next_row else evals[:6]) + (self.qin_eval, self.z3_shifted_eval)

    def round_5(self):
        n, pk = self.group_order, self.pk
        zeta, v = self.zeta, self.v
        al, be, ga = self.alpha, self.beta, self.gamma
        a, b, c = self.a_eval, self.b_eval, self.c_eval
        s1, s2, zw = self.s1_eval, self.s2_eval, self.z_shifted_eval
        aw, bw, cw = self.shifted
        qin, z3w = self.qin_eval, self.z3_shifted_eval
        zn = pow(zeta, n, R)
        ZH_ev = (zn - 1) % R
        L0_ev = ZH_ev * O.inv0(n * (zeta - 1), R) % R
        PI_ev = O.barycentric_eval(self.PI, zeta)
        c1 = (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al % R
        c2 = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
        al2l0 = al * al % R * L0_ev % R
        al3, al4 = pow(al, 3, R), pow(al, 4, R)
        K = (self.kappa + a + self.theta * b + self.theta * self.theta % R * c - 1) % R
        qc = list(pk.QC)
        for e, col in pk.custom:  # the terms at the evaluations: a constant selector, like QC
            m = NR.monomial(e, (a, b, c, aw, bw, cw))
            qc = [(x + m * y) % R for x, y in zip(qc, col)]
        QL, QR, QM, QO, QC, S1, S2, S3, QIN, QOUT = (O.ifft(p) for p in (pk.QL, pk.QR, pk.QM, pk.QO, qc, pk.S1, pk.S2,
                                                                        pk.S3, pk.q_in, pk.q_out))
        v2, v3, v4, v5, v6 = (pow(v, e, R) for e in (2, 3, 4, 5, 6))
        num = ZO.lincomb([(QL, a), (QR, b), (QM, a * b), (QO, c), (QC, 1), (self.Zb, c1 + al2l0), (S3, -c2 * be),
                          (self.T1b, -ZH_ev), (self.T2b, -ZH_ev * zn), (self.T3b, -ZH_ev * zn * zn),
                          (self.Ab, v), (self.Bb, v2), (self.Cb, v3), (S1, v4), (S2, v5),
                          (QOUT, al3 * z3w % R * K), (self.Z3c, -al3 * (1 + qin * K) + al4 * L0_ev), (QIN, v6)], n + 9)
        num[0] = (num[0] + PI_ev - c2 * (c + ga) - al2l0 - v * a - v2 * b - v3 * c - v4 * s1 - v5 * s2
                  + al3 * z3w - al4 * L0_ev - v6 * qin) % R
        Wz = ZO.divide_linear(num, zeta)
        if self.next_row:  # Z, A, B, C, then Z3 at v^4
            numw = ZO.lincomb([(self.Zb, 1), (self.Ab, v), (self.Bb, v2), (self.Cb, v3), (self.Z3c, v4)], n + 3)
            numw[0] = (numw[0] - zw - v * aw - v2 * bw - v3 * cw - v4 * z3w) % R
        else:
            numw = ZO.lincomb([(self.Zb, 1), (self.Z3c, v)], n + 3)
            numw[0] = (numw[0] - zw - v * z3w) % R
        Wzw = ZO.divide_linear(numw, zeta * O.root_of_unity(n) % R)
        return NR._commit(self.setup, Wz), NR._commit(self.setup, Wzw)


def prove(setup, pk: ShufflePreprocessed, A, B, C, public_inputs, fast: bool = False, check: bool = True) -> dict:
    """the oracle's proof of a circuit with a shuffle; ``fast``: transforms by the C restatement (setup: an
    oracle.fast.Setup)"""
    if fast:
        with F.c_kernels():
            return ShuffleProver(setup, pk, check=check).prove(A, B, C, public_inputs)
    return ShuffleProver(setup, pk, check=check).prove(A, B, C, public_inputs)


def proof_bytes(proof: dict) -> bytes:
    """768 plain bytes, the shifted wire evaluations of a next-row proof, z3_1, qin_eval, z3_shifted_eval"""
    out = O.proof_bytes(proof)
    if "a_shifted_eval" in proof:
        out += b"".join(int(proof[k]).to_bytes(32, "big") for k in NR.NEXT_ROW_FIELDS)
    x, y = proof["z3_1"]
    return out + b"".join(int(t).to_bytes(32, "big") for t in (x, y, proof["qin_eval"], proof["z3_shifted_eval"]))


def challenges(proof: dict, next_row: bool) -> dict:
    """the shuffle transcript (plonkathon_b200/transcript.py SHUFFLE_SCHEDULE), restated on the oracle's transcript"""
    tr = O.Transcript(b"plonk")
    steps = [(("a_1", "b_1", "c_1"), ("beta", "gamma", "theta", "kappa")), (("z_1", "z3_1"), ("alpha", "fft_cofactor")),
             (("t_lo_1", "t_mid_1", "t_hi_1"), ("zeta",)), (round4_fields(next_row), ("v",)),
             (("W_z_1", "W_zw_1"), ("u",))]
    out = {}
    for fields, drawn in steps:
        for f in fields:
            (tr.append_point if isinstance(proof[f], tuple) else tr.append_scalar)(f.encode(), proof[f])
        for lbl in drawn:
            out[lbl] = tr.get_and_append_challenge(lbl.encode())
    return out


def verify_proof_trapdoor(group_order: int, vk: dict, custom_pts, shuffle_pts, proof: dict, public, tau: int) -> bool:
    """the batched verifier of a shuffle proof with the final pairing equation checked through tau.  custom_pts:
    (exponents, [Q_k]) in the prover's order; shuffle_pts: ([q_in], [q_out]), None for a zero column"""
    n = group_order
    next_row = "a_shifted_eval" in proof
    ch = challenges(proof, next_row)
    be, ga, al, zeta, v, u = ch["beta"], ch["gamma"], ch["alpha"], ch["zeta"], ch["v"], ch["u"]
    th, ka = ch["theta"], ch["kappa"]
    w = O.root_of_unity(n)
    ZH = (pow(zeta, n, R) - 1) % R
    L0 = ZH * O.inv0(n * (zeta - 1), R) % R
    PI = sum((-p) * pow(w, i, R) % R * ZH % R * O.inv0(n * (zeta - pow(w, i, R)), R) for i, p in enumerate(public)) % R
    a, b, c = proof["a_eval"], proof["b_eval"], proof["c_eval"]
    s1, s2, zw = proof["s1_eval"], proof["s2_eval"], proof["z_shifted_eval"]
    aw, bw, cw = (proof[k] for k in NR.NEXT_ROW_FIELDS) if next_row else (0, 0, 0)
    qin, z3w = proof["qin_eval"], proof["z3_shifted_eval"]
    a2 = al * al % R
    a3, a4 = a2 * al % R, a2 * a2 % R
    v2, v3, v4, v5, v6 = (pow(v, k, R) for k in range(2, 7))
    K = (ka + a + th * b + th * th % R * c - 1) % R
    vz3 = v4 if next_row else v
    sig = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
    r0 = (PI - L0 * a2 - sig * (c + ga) + a3 * z3w - a4 * L0) % R
    nr = u if next_row else 0  # A, B, C join the zeta w batch on a next-row circuit
    pts = [
        (vk["Qm"], a * b), (vk["Ql"], a), (vk["Qr"], b), (vk["Qo"], c), (vk["Qc"], 1),
        *[(p, NR.monomial(e, (a, b, c, aw, bw, cw))) for e, p in custom_pts],
        (proof["z_1"], (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al
         + L0 * a2 + u),
        (vk["S3"], -sig * be),
        (proof["t_lo_1"], -ZH), (proof["t_mid_1"], -ZH * pow(zeta, n, R)), (proof["t_hi_1"], -ZH * pow(zeta, 2 * n, R)),
        (proof["a_1"], v + nr * v), (proof["b_1"], v2 + nr * v2), (proof["c_1"], v3 + nr * v3),
        (vk["S1"], v4), (vk["S2"], v5),
        (shuffle_pts[1], a3 * z3w % R * K), (proof["z3_1"], -a3 * (1 + qin * K) + a4 * L0 + u * vz3),
        (shuffle_pts[0], v6),
    ]
    Fp = O.ec_lincomb_naive([(p, k % R) for p, k in pts if p is not None])
    E = (-r0 + v * a + v2 * b + v3 * c + v4 * s1 + v5 * s2 + v6 * qin
         + u * (zw + v * aw + v2 * bw + v3 * cw + vz3 * z3w)) % R
    lhs = O.g1_multiply(O.ec_lincomb_naive([(proof["W_z_1"], 1), (proof["W_zw_1"], u)]), tau)
    rhs = O.ec_lincomb_naive([(proof["W_z_1"], zeta), (proof["W_zw_1"], u * zeta % R * w), (Fp, 1), (O.G1, -E % R)])
    return lhs == rhs


def preprocessed(c, S=None) -> ShufflePreprocessed:
    """ShufflePreprocessed of a plonkathon_b200.synthetic.ArrayCircuit with a shuffle"""
    base = CG.preprocessed(c, S)
    q_in, q_out = c.shuffle
    return ShufflePreprocessed(*[getattr(base, f) for f in base.__dataclass_fields__], list(q_in), list(q_out))
