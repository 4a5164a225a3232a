"""Drop-in for the reference's ``verifier.py``: ``VerificationKey`` (verifier.py:10-37) with the two
verification routines the reference leaves as stubs (verifier.py:40-92; their completed form is what
``test.py:115-133`` runs as ``TestingVerificationKey``) and ``compute_challenges`` (verifier.py:95-106).

The G1 linear combinations go through ``ec_lincomb`` (GPU MSM), G2 arithmetic and the pairing through the
library's host code (csrc/pairing.cuh).  Each pairing equation  e(L, [1]_2) == e(W, Q)  is checked as
e(L, [1]_2) * e(-W, Q) == 1 -- a product of two Miller loops and one final exponentiation.

Notation follows the PLONK paper's verifier: zeta evaluation point, v batching challenge, u the challenge
that merges the two opening checks, bars for the prover-supplied evaluations."""
from __future__ import annotations

from dataclasses import dataclass

from .curve import G1, G2, Scalar, ec_lincomb, g1_neg, g2_add, g2_mul, pairing_product_is_one
from . import _lib
from .custom_gates import is_next_row, monomial
from .field import CURVE_ORDER, FIELD_MODULUS
from .transcript import Transcript


def _lagrange_terms_at(group_order: int, values, x: Scalar) -> Scalar:
    """sum_i values[i] * L_i(x) for the first len(values) Lagrange polynomials of the domain:
    L_i(x) = w^i (x^n - 1) / (n (x - w^i)).  Equal to Polynomial(values + zeros, LAGRANGE).barycentric_eval(x)
    (poly.py:181-195; division by zero yields zero there as here) without materialising n - len(values) zeros."""
    w = Scalar.root_of_unity(group_order)
    zh = x ** group_order - 1
    acc, wi = Scalar(0), Scalar(1)
    for val in values:
        acc += Scalar(val) * wi * zh / ((x - wi) * group_order)
        wi *= w
    return acc


@dataclass
class VerificationKey:
    """verifier.py:10-37."""
    group_order: int
    Qm: object
    Ql: object
    Qr: object
    Qo: object
    Qc: object
    S1: object
    S2: object
    S3: object
    X_2: object
    w: Scalar
    # custom gate terms ((i, j, l) or (i, j, l, i', j', l'), commitment to Q_k), in the prover's order
    # (plonkathon_b200/custom_gates.py); with a next-row term the key takes NextRowProof only
    custom: tuple = ()
    # lookup argument (plonkathon_b200/lookup.py): ([q_K], [t1], [t2], [t3]) for one table, ([q_K], [t1], [t2], [t3],
    # [Q_T], [t4]) for several tables told apart by a tag; the identity (None) for a zero column; () without lookups
    lookup: tuple = ()
    # shuffle (plonkathon_b200/shuffle.py): ([q_in], [q_out]), the identity (None) for a zero column; () without one.
    # With a shuffle the key takes ShuffleProof only (NextRowShuffleProof with a next-row term)
    shuffle: tuple = ()

    def _custom_terms(self, a, b, c, aw=None, bw=None, cw=None):
        """the custom gates' part of the linearisation: sum_k m_k(a, b, c, a(zeta w), b(zeta w), c(zeta w)) [Q_k]"""
        return [(pt, monomial(e, a, b, c, aw, bw, cw)) for e, pt in self.custom]

    @property
    def next_row(self) -> bool:
        """whether some custom term reads the next row"""
        return any(is_next_row(e) for e, _ in self.custom)

    @staticmethod
    def _well_formed(pf) -> bool:
        """every commitment of the proof is a point of the curve y^2 = x^3 + 3 with reduced coordinates and every
        evaluation is a reduced scalar: a malformed proof is rejected (False), it must not reach the MSM"""
        for v in pf.flatten().values():
            if isinstance(v, tuple):
                x, y = int(v[0]), int(v[1])
                if not (0 <= x < FIELD_MODULUS and 0 <= y < FIELD_MODULUS and (y * y - x * x * x - 3) % FIELD_MODULUS == 0):
                    return False
            elif v is None or not 0 <= int(v) < CURVE_ORDER:
                return False
        return True

    @property
    def _kind(self):
        """the proof kind of the key's blocks (prover.KINDS), None for a combination without one"""
        from .prover import proof_kind
        return proof_kind(next_row=self.next_row, shuffle=bool(self.shuffle), lookup=bool(self.lookup))

    def _matches(self, pf) -> bool:
        """the key takes the proofs of its kind only: a plain key plain proofs, a lookup key lookup proofs, ..."""
        kind = self._kind
        return kind is not None and isinstance(pf, kind.proof)

    def verify_proof(self, group_order: int, pf, public=[]) -> bool:
        """verifier.py:40-73: the batched form -- one pairing equation, the linearisation commitment never
        formed on its own.  Malformed proofs (points off the curve, the identity) are rejected, not raised; so is a
        plain proof against a lookup key and the reverse."""
        if not self._matches(pf) or not self._well_formed(pf):
            return False
        try:
            return self._verify(group_order, pf, public, batched=True)
        except _lib.PlonkB200Error:
            return False

    def verify_proof_unoptimized(self, group_order: int, pf, public=[]) -> bool:
        """verifier.py:76-92: rebuild the commitment to the prover's linearisation polynomial R (R(zeta) == 0),
        then check the opening at zeta and the opening of Z at zeta*w separately."""
        if not self._matches(pf) or not self._well_formed(pf):
            return False
        try:
            return self._verify(group_order, pf, public, batched=False)
        except _lib.PlonkB200Error:
            return False

    # ---- both routines, plain and lookup proofs: steps 4-12 of the paper's verifier
    def _verify(self, group_order: int, pf, public, batched: bool) -> bool:
        n = group_order
        proof = pf.flatten()
        ch = Transcript(b"plonk").replay(self._kind.schedule, proof)
        beta, gamma, alpha, zeta, v, u = ch["beta"], ch["gamma"], ch["alpha"], ch["zeta"], ch["v"], ch["u"]
        zh_ev = zeta ** n - 1
        l0_ev = zh_ev / ((zeta - 1) * n)
        pi_ev = _lagrange_terms_at(n, [-int(x) % CURVE_ORDER for x in public], zeta)
        a, b, c = proof["a_eval"], proof["b_eval"], proof["c_eval"]
        s1, s2, zw = proof["s1_eval"], proof["s2_eval"], proof["z_shifted_eval"]
        # the wires at zeta w (next-row keys only)
        aw, bw, cw = (proof.get(k) for k in ("a_shifted_eval", "b_shifted_eval", "c_shifted_eval"))
        root = Scalar.root_of_unity(n)
        zeta_n = zeta ** n
        a2 = alpha * alpha
        v2, v3, v4, v5 = v ** 2, v ** 3, v ** 4, v ** 5
        sigma_bar = (a + beta * s1 + gamma) * (b + beta * s2 + gamma) * zw
        # the linearisation R without its constant, and the constant r0 (R(zeta) == 0)
        r_terms = [
            (self.Qm, a * b), (self.Ql, a), (self.Qr, b), (self.Qo, c), (self.Qc, 1), *self._custom_terms(a, b, c, aw, bw, cw),
            (proof["z_1"], (a + beta * zeta + gamma) * (b + beta * 2 * zeta + gamma) * (c + beta * 3 * zeta + gamma)
             * alpha + l0_ev * a2),
            (self.S3, -sigma_bar * alpha * beta),
            (proof["t_lo_1"], -zh_ev), (proof["t_mid_1"], -zh_ev * zeta_n), (proof["t_hi_1"], -zh_ev * zeta_n * zeta_n),
        ]
        r0 = pi_ev - l0_ev * a2 - sigma_bar * alpha * (c + gamma)
        # the openings at zeta and at zeta w: (commitment, batching weight), and the claimed value of each batch
        at_zeta = [(proof["a_1"], v), (proof["b_1"], v2), (proof["c_1"], v3), (self.S1, v4), (self.S2, v5)]
        e_zeta = v * a + v2 * b + v3 * c + v4 * s1 + v5 * s2
        at_zw = [(proof["z_1"], Scalar(1))]
        e_zw = zw
        if self.next_row:  # A, B, C join Z at zeta w: v (A - a(zeta w)) + v^2 (B - b(zeta w)) + v^3 (C - c(zeta w))
            at_zw += [(proof["a_1"], v), (proof["b_1"], v2), (proof["c_1"], v3)]
            e_zw = e_zw + v * aw + v2 * bw + v3 * cw
        if self.lookup:
            eta, delta, eps = ch["eta"], ch["delta"], ch["epsilon"]
            fe, te, tw = proof["f_eval"], proof["t_eval"], proof["t_shifted_eval"]
            h2e, h1w, z2w = proof["h2_eval"], proof["h1_shifted_eval"], proof["z2_shifted_eval"]
            a3, a4 = a2 * alpha, a2 * a2
            a5 = a4 * alpha
            od = delta + 1
            eod = eps * od
            hw = eod + h2e + delta * h1w
            # several tables: ([q_K], [t1], [t2], [t3], [Q_T], [t4]); one table: the first four
            qk, t1, t2, t3, *tag = self.lookup
            eta3 = eta * eta * eta
            t_parts = [(t1, Scalar(1)), (t2, eta), (t3, eta * eta)]  # [T] = [t1] + eta [t2] + eta^2 [t3] (+ eta^3 [t4])
            if tag:
                qt, t4 = tag
                r_terms.append((qt, a3 * eta3))  # alpha^3 eta^3 Q_T
                t_parts.append((t4, eta3))
            r_terms += [
                # alpha^3 q_K (a + eta b + eta^2 c - f)
                (qk, a3 * (a + eta * b + eta * eta * c - fe)),
                # alpha^4 [Z2 (1+d)(e+f)(e(1+d) + t + d t_w) - z2_w (e(1+d) + H1 + d h2) hw] + alpha^5 L0 (Z2 - 1)
                (proof["z2_1"], a4 * od * (eps + fe) * (eod + te + delta * tw) + a5 * l0_ev),
                (proof["h1_1"], -a4 * z2w * hw),
            ]
            r0 = r0 - a4 * z2w * (eod + delta * h2e) * hw - a5 * l0_ev
            v6, v7, v8 = v5 * v, v5 * v2, v5 * v3
            at_zeta += [(proof["f_1"], v6), (proof["h2_1"], v8)] + [(p, k * v7) for p, k in t_parts]
            e_zeta = e_zeta + v6 * fe + v7 * te + v8 * h2e
            at_zw += [(proof["h1_1"], v2), (proof["z2_1"], v3)] + [(p, k * v) for p, k in t_parts]
            e_zw = e_zw + v * tw + v2 * h1w + v3 * z2w
        if self.shuffle:
            theta, kappa = ch["theta"], ch["kappa"]
            qin, z3w = proof["qin_eval"], proof["z3_shifted_eval"]
            a3, a4 = a2 * alpha, a2 * a2
            k = kappa + a + theta * b + theta * theta * c - 1  # kappa + w - 1
            qin_pt, qout_pt = self.shuffle
            r_terms += [
                # alpha^3 [z3_w (1 + Q_out k) - Z3 (1 + q_in k)] + alpha^4 L0 (Z3 - 1)
                (qout_pt, a3 * z3w * k),
                (proof["z3_1"], -a3 * (qin * k + 1) + a4 * l0_ev),
            ]
            r0 = r0 + a3 * z3w - a4 * l0_ev
            v6 = v5 * v
            at_zeta.append((qin_pt, v6))
            e_zeta = e_zeta + v6 * qin
            vk = v4 if self.next_row else v  # after A, B, C at zeta w on a next-row key
            at_zw.append((proof["z3_1"], vk))
            e_zw = e_zw + vk * z3w
        if batched:
            # e(W_z + u W_zw, [x]_2) == e(zeta W_z + u zeta w W_zw + F - E, [1]_2), F = [R] - r0 + both batches
            f_pt = ec_lincomb(r_terms + at_zeta + [(p, u * k) for p, k in at_zw])
            e_scalar = -r0 + e_zeta + u * e_zw
            lhs = ec_lincomb([(proof["W_z_1"], 1), (proof["W_zw_1"], u)])
            rhs = ec_lincomb([(proof["W_z_1"], zeta), (proof["W_zw_1"], u * zeta * root), (f_pt, 1), (G1, -e_scalar)])
            return pairing_product_is_one([(lhs, self.X_2), (g1_neg(rhs), G2)])
        # R's commitment formed, then the opening at zeta and the opening at zeta w, each its own pairing product
        batch = ec_lincomb(r_terms + [(G1, r0)] + at_zeta + [(G1, -e_zeta)])
        x_minus_zeta = g2_add(self.X_2, g2_mul(G2, -zeta))
        if not pairing_product_is_one([(batch, G2), (g1_neg(proof["W_z_1"]), x_minus_zeta)]):
            return False
        shifted = ec_lincomb(at_zw + [(G1, -e_zw)])
        x_minus_zeta_w = g2_add(self.X_2, g2_mul(G2, -(zeta * root)))
        return pairing_product_is_one([(shifted, G2), (g1_neg(proof["W_zw_1"]), x_minus_zeta_w)])

    def compute_challenges(self, proof):
        """verifier.py:95-106: replay the prover's transcript over the proof's five messages."""
        transcript = Transcript(b"plonk")
        beta, gamma = transcript.round_1(proof.msg_1)
        alpha, _fft_cofactor = transcript.round_2(proof.msg_2)
        zeta = transcript.round_3(proof.msg_3)
        v = transcript.round_4(proof.msg_4)
        u = transcript.round_5(proof.msg_5)
        return beta, gamma, alpha, zeta, v, u
