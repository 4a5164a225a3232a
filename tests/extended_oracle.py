"""TEST INFRASTRUCTURE ONLY -- the oracle prover and trapdoor verifier of every proof kind.

oracle/plonk_oracle.py restates the reference's plain PLONK and stays pinned by the reference's fixtures.  The reference
has none of the features below, so this module extends it, reusing its transforms (``to_coset_extended_lagrange``,
``coset_extended_lagrange_to_coeffs``, ``barycentric_eval``) and its transcript, and states each piece once:
  * custom gate terms: the gate gains sum_k Q_k a^i b^j c^l a(wX)^i' b(wX)^j' c(wX)^l' (plonkathon_b200/custom_gates.py,
    three exponents for a same-row term).  A term over the next row makes the proof a next-row proof: A, B, C are also
    opened at zeta w;
  * a shuffle (plonkathon_b200/shuffle.py): the q_in rows and the q_out rows hold the same multiset of (a, b, c).  With
    w = a + theta b + theta^2 c, Z3_(i+1) = Z3_i (1 + q_in (kappa + w - 1)) / (1 + q_out (kappa + w - 1));
  * a lookup argument: plookup (eprint 2020/315) in PlonKup's cyclic, alternating-split form (eprint 2022/086) over
    the concatenated tables, a row matching (a, b, c, Q_T) against (t1, t2, t3, t4).  One table is Q_T = t4 = 0;
  * zero knowledge (the PLONK paper, eprint 2019/953, rounds 1-3): each committed polynomial P becomes
    P + (b_s X^(k-1) + ... + b_(s+k-1)) Z_H with the positions of BLINDERS, and the quotient T, cut at n and 2n, becomes
    T1' = T1 + b10 X^n, T2' = T2 - b10 + b11 X^n, T3' = T3 - b11.
Every committed polynomial is kept in coefficient form and committed as such; without blinders the commitments are
those of the unblinded polynomials.  The quotient is one sum on the 4n coset, and round 5 one linearisation, which the
trapdoor verifier evaluates over the commitments.  DESIGN.md fixes the algebra of each argument.  Running inside
``oracle.fast.c_kernels()`` (``prove(..., fast=True)``) answers the transforms with the C restatement."""
from __future__ import annotations

from dataclasses import dataclass, field

from oracle import c_oracle as CO
from oracle import fast as F
from oracle import plonk_oracle as O

R = O.R_MOD
BLOCKS = ("plain", "next_row", "shuffle", "lookup")
STEPS = ("1", "1L", "2", "3", "4", "5")

# the proof's fields per block and transcript step, in the order the proof and the transcript hold them
FIELDS = {
    "plain": {"1": ("a_1", "b_1", "c_1"), "2": ("z_1",), "3": ("t_lo_1", "t_mid_1", "t_hi_1"),
              "4": ("a_eval", "b_eval", "c_eval", "s1_eval", "s2_eval", "z_shifted_eval"), "5": ("W_z_1", "W_zw_1")},
    "next_row": {"4": ("a_shifted_eval", "b_shifted_eval", "c_shifted_eval")},
    "shuffle": {"2": ("z3_1",), "4": ("qin_eval", "z3_shifted_eval")},
    "lookup": {"1L": ("f_1", "h1_1", "h2_1"), "2": ("z2_1",),
               "4": ("f_eval", "t_eval", "t_shifted_eval", "h2_eval", "h1_shifted_eval", "z2_shifted_eval")},
}
# the challenges each block draws after a step's fields
CHALLENGES = {
    "plain": {"1": ("beta", "gamma"), "2": ("alpha", "fft_cofactor"), "3": ("zeta",), "4": ("v",), "5": ("u",)},
    "next_row": {},
    "shuffle": {"1": ("theta", "kappa")},
    "lookup": {"1": ("eta",), "1L": ("delta", "epsilon")},
}

# kind (its blocks after "plain") -> (m, positions of b1..bm in the flat list the product's set_zk, set_zk_shuffle or
# set_zk_lookup takes, per blinded polynomial, highest power of X first); "T" holds b10, b11 of the quotient split
_ZK = {"A": (0, 1), "B": (2, 3), "C": (4, 5), "Z": (6, 7, 8), "T": (9, 10)}
_ZK_NEXT = dict(_ZK, A=(11, 0, 1), B=(12, 2, 3), C=(13, 4, 5))
BLINDERS = {
    (): (11, _ZK),
    ("next_row",): (14, _ZK_NEXT),
    ("shuffle",): (14, dict(_ZK, Z3=(11, 12, 13))),
    ("next_row", "shuffle"): (17, dict(_ZK_NEXT, Z3=(14, 15, 16))),
    ("lookup",): (21, dict(_ZK, F=(11, 12), H1=(13, 14, 15), H2=(16, 17), Z2=(18, 19, 20))),
}

NOT_A_SHUFFLE = "shuffle: the q_in rows and the q_out rows are not permutations of each other"


@dataclass
class Preprocessed(O.Preprocessed):
    custom: list = field(default_factory=list)  # ((3 or 6 exponents), n Lagrange values of Q_k)
    q_in: list = None   # the shuffle's selectors, n values 0 / 1
    q_out: list = None
    qk: list = None     # the lookup selector, n values 0 / 1
    table: list = None  # [t1, t2, t3] over the concatenated tables, padded to n by repeating the last row
    qtag: list = None   # Q_T: the table id of each lookup row, 0 elsewhere
    t4: list = None     # each table row's id, padded as the table


def kind(pk) -> tuple:
    """the blocks of pk's proofs after "plain" """
    on = {"next_row": any(any(e[3:]) for e, _ in pk.custom), "shuffle": pk.q_in is not None,
          "lookup": pk.qk is not None}
    return tuple(b for b in BLOCKS[1:] if on[b])


def blinder_count(pk) -> int:
    return BLINDERS[kind(pk)][0]


def preprocessed(c, S=None) -> Preprocessed:
    """Preprocessed of a plonkathon_b200.synthetic.ArrayCircuit"""
    from plonkathon_b200 import synthetic as syn
    from plonkathon_b200.lookup import check_lookups, padded_table
    n = c.group_order
    S1, S2, S3 = S or syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    pk = Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, S1, S2, S3, list(c.custom))
    if c.shuffle:
        pk.q_in, pk.q_out = (list(q) for q in c.shuffle)
    if c.lookup or c.lookups:
        pk.qk, pk.qtag, cols, _ = check_lookups(c.lookups or [c.lookup], n)
        *pk.table, pk.t4 = padded_table(cols, n)
    return pk


# ---- polynomials in coefficient form -------------------------------------------------------------------------------
def monomial(exps, vals) -> int:
    """m_k over (a, b, c, a(wX), b(wX), c(wX)); three exponents for a same-row term"""
    m = 1
    for x, e in zip(vals, exps):
        if e:
            m = m * pow(x, e, R) % R
    return m


def poly_eval(coeffs, x):
    acc = 0
    for c in reversed(coeffs):
        acc = (acc * x + c) % R
    return acc


def add_zh_multiple(coeffs, c, n):
    """coeffs (zero padded to n + len(c)) + (c[0] + c[1] X + ...) (X^n - 1)"""
    out = [int(x) % R for x in coeffs] + [0] * (n + len(c) - len(coeffs))
    for i, ci in enumerate(c):
        out[i] = (out[i] - ci) % R
        out[n + i] = (out[n + i] + ci) % R
    return out


def divide_linear(num, point):
    """num / (X - point) by synthetic division; asserts the remainder is zero"""
    q = [0] * (len(num) - 1)
    acc = 0
    for i in range(len(num) - 1, 0, -1):
        acc = (acc * point + num[i]) % R
        q[i - 1] = acc
    assert (acc * point + num[0]) % R == 0, "opening numerator is not divisible by (X - point)"
    return q


def lincomb(terms):
    out = [0] * max(len(p) for p, _ in terms)
    for vec, w in terms:
        w %= R
        if w:
            for i, x in enumerate(vec):
                out[i] = (out[i] + w * x) % R
    return out


def commit_coeffs(setup, coeffs):
    """[sum_i c_i tau^i] G, trailing zero coefficients left out (they need no SRS power); setup: a plonk_oracle.Setup
    or an oracle.fast.Setup"""
    c = [int(x) % R for x in coeffs]
    while len(c) > 1 and c[-1] == 0:
        c.pop()
    if len(c) > (setup.pts.shape[0] if isinstance(setup, F.Setup) else len(setup.powers_of_x)):
        raise Exception("Not enough powers in setup")
    if isinstance(setup, F.Setup):
        return CO.g1_lincomb(setup.pts[:len(c)], F._to_np(c))
    return setup.commit_coeffs(c)


def gate(Q, PI, custom, A, B, C, s):
    """the gate constraint at every point of a domain: Q = (QL, QR, QM, QO, QC), PI, custom = [(exps, Q_k)] and the
    wires as values there; s: the index step of X -> wX (1 on H, 4 on the 4n coset)"""
    QL, QR, QM, QO, QC = Q
    m = len(A)
    out = []
    for j in range(m):
        a, b, c, j1 = A[j], B[j], C[j], (j + s) % m
        vals = (a, b, c, A[j1], B[j1], C[j1])
        out.append((a * QL[j] + b * QR[j] + a * b % R * QM[j] + c * QO[j] + PI[j] + QC[j]
                    + sum(q[j] * monomial(e, vals) for e, q in custom)) % R)
    return out


def linearisation(blocks, n, ch, ev, pi, P):
    """R(X) = sum_i w_i P_i(X) + r0, which vanishes at zeta, and the two opening batches, over the polynomials ``P``
    (name -> coefficients for the prover, name -> commitment for the verifier) -> (terms [(P_i, w_i)], r0,
    [(P, value)] opened at zeta, [(P, value)] opened at zeta w)"""
    al, be, ga, zeta = ch["alpha"], ch["beta"], ch["gamma"], ch["zeta"]
    a, b, c = ev["a_eval"], ev["b_eval"], ev["c_eval"]
    s1, s2, zw = ev["s1_eval"], ev["s2_eval"], ev["z_shifted_eval"]
    shifted = tuple(ev.get(k, 0) for k in FIELDS["next_row"]["4"])
    zn = pow(zeta, n, R)
    ZH = (zn - 1) % R
    L0 = ZH * O.inv0(n * (zeta - 1), R) % R
    al2, al3 = al * al % R, pow(al, 3, R)
    al4, al5 = al3 * al % R, pow(al, 5, R)
    perm = (a + be * zeta + ga) * (b + 2 * be * zeta + ga) % R * (c + 3 * be * zeta + ga) % R * al % R
    sig = (a + be * s1 + ga) * (b + be * s2 + ga) % R * al % R * zw % R
    terms = [(P["Ql"], a), (P["Qr"], b), (P["Qm"], a * b), (P["Qo"], c), (P["Qc"], 1)]
    terms += [(q, monomial(e, (a, b, c) + shifted)) for e, q in P["custom"]]
    terms += [(P["Z"], perm + al2 * L0), (P["S3"], -sig * be),
              (P["T1"], -ZH), (P["T2"], -ZH * zn), (P["T3"], -ZH * zn * zn)]
    r0 = pi - sig * (c + ga) - al2 * L0
    at_z = [(P["A"], a), (P["B"], b), (P["C"], c), (P["S1"], s1), (P["S2"], s2)]
    at_zw = [(P["Z"], zw)]
    if "next_row" in blocks:
        at_zw += [(P["A"], shifted[0]), (P["B"], shifted[1]), (P["C"], shifted[2])]
    if "shuffle" in blocks:
        th, qin, z3w = ch["theta"], ev["qin_eval"], ev["z3_shifted_eval"]
        K = (ch["kappa"] + a + th * b + th * th % R * c - 1) % R
        terms += [(P["Qout"], al3 * z3w % R * K), (P["Z3"], -al3 * (1 + qin * K) + al4 * L0)]
        r0 += al3 * z3w - al4 * L0
        at_z.append((P["Qin"], qin))
        at_zw.append((P["Z3"], z3w))
    if "lookup" in blocks:
        eta, d, e = ch["eta"], ch["delta"], ch["epsilon"]
        fe, te, tw = ev["f_eval"], ev["t_eval"], ev["t_shifted_eval"]
        h2e, h1w, z2w = ev["h2_eval"], ev["h1_shifted_eval"], ev["z2_shifted_eval"]
        od, eod = (1 + d) % R, e * (1 + d) % R
        hw = (eod + h2e + d * h1w) % R
        terms += [(P["Qk"], al3 * ((a + eta * b + eta * eta % R * c - fe) % R)), (P["Qt"], al3 * pow(eta, 3, R)),
                  (P["Z2"], al4 * od % R * (e + fe) % R * ((eod + te + d * tw) % R) + al5 * L0),
                  (P["H1"], -al4 * z2w % R * hw)]
        r0 -= al4 * z2w % R * ((eod + d * h2e) % R) % R * hw + al5 * L0
        at_z += [(P["F"], fe), (P["T"], te), (P["H2"], h2e)]
        at_zw += [(P["T"], tw), (P["H1"], h1w), (P["Z2"], z2w)]
    return terms, r0 % R, at_z, at_zw


# ---- the proof and its transcript ----------------------------------------------------------------------------------
def proof_fields(blocks=()) -> tuple:
    return tuple(f for b in ("plain",) + tuple(blocks) for s in STEPS for f in FIELDS[b].get(s, ()))


def proof_kind(proof: dict) -> tuple:
    return tuple(b for b in BLOCKS[1:] if FIELDS[b]["4"][0] in proof)


def proof_bytes(proof: dict) -> bytes:
    out = bytearray()
    for k in proof_fields(proof_kind(proof)):
        v = proof[k]
        out += b"".join(int(x).to_bytes(32, "big") for x in (v if isinstance(v, tuple) else (v,)))
    return bytes(out)


def proof_from_bytes(raw: bytes) -> dict:
    """the proof of the kind whose size is len(raw)"""
    for blocks in BLINDERS:
        fields = proof_fields(blocks)
        words = [int.from_bytes(raw[i:i + 32], "big") for i in range(0, len(raw), 32)]
        if 32 * sum(1 + f.endswith("_1") for f in fields) == len(raw):
            out = {}
            for f in fields:
                out[f] = (words.pop(0), words.pop(0)) if f.endswith("_1") else words.pop(0)
            return out
    raise ValueError("no proof kind has %d bytes" % len(raw))


def _step(tr, blocks, step, proof) -> dict:
    """absorbs a step's fields of ``proof`` and draws its challenges"""
    blocks = ("plain",) + tuple(blocks)
    for b in blocks:
        for f in FIELDS[b].get(step, ()):
            (tr.append_point if isinstance(proof[f], tuple) else tr.append_scalar)(f.encode(), proof[f])
    return {c: tr.get_and_append_challenge(c.encode()) for b in blocks for c in CHALLENGES[b].get(step, ())}


def challenges(proof: dict) -> dict:
    tr, blocks, out = O.Transcript(b"plonk"), proof_kind(proof), {}
    for s in STEPS:
        if any(s in FIELDS[b] for b in ("plain",) + blocks):
            out.update(_step(tr, blocks, s, proof))
    return out


# ---- the prover ----------------------------------------------------------------------------------------------------
class Prover:
    def __init__(self, setup, pk: Preprocessed, blinders=None, check: bool = True):
        self.setup, self.pk, self.n, self.check = setup, pk, pk.group_order, check
        self.blocks = kind(pk)
        count, self.layout = BLINDERS[self.blocks]
        self.blinders = [0] * count if blinders is None else [int(x) % R for x in blinders]
        assert len(self.blinders) == count

    def _zh(self, name):
        """the Z_H multiple of polynomial ``name``, lowest coefficient first"""
        return [self.blinders[i] for i in reversed(self.layout[name])]

    def _blind(self, name, values):
        return add_zh_multiple(O.ifft(values), self._zh(name), self.n)

    def _ext(self, values):
        return O.to_coset_extended_lagrange(values, self.fft_cofactor)

    def prove(self, A, B, C, public_inputs) -> dict:
        n, tr, proof = self.n, O.Transcript(b"plonk"), {}
        self.PI = [(-int(v)) % R for v in public_inputs] + [0] * (n - len(public_inputs))
        rounds = {"1": lambda: self.round_1(A, B, C), "1L": self.round_1L, "2": self.round_2, "3": self.round_3,
                  "4": self.round_4, "5": self.round_5}
        for s in STEPS:
            if s == "1L" and "lookup" not in self.blocks:
                continue
            proof.update(rounds[s]())
            for k, x in _step(tr, self.blocks, s, proof).items():
                setattr(self, k, x)
        return proof

    def round_1(self, A, B, C):
        """the witness checks: gates (row i + 1 for next-row terms), the shuffle's multisets, the table membership"""
        n, pk = self.n, self.pk
        self.A, self.B, self.C = W = [[int(v) % R for v in X] + [0] * (n - len(X)) for X in (A, B, C)]
        if self.check:
            g = gate((pk.QL, pk.QR, pk.QM, pk.QO, pk.QC), self.PI, pk.custom, *W, 1)
            for i in range(n):
                assert g[i] == 0, "gate %d unsatisfied" % i
        if "shuffle" in self.blocks:
            side = lambda q: sorted(tuple(c[i] for c in W) for i in range(n) if q[i])  # noqa: E731
            assert side(pk.q_in) == side(pk.q_out), NOT_A_SHUFFLE
        if "lookup" in self.blocks:
            idx = {}
            for j, row in enumerate(zip(*pk.table, pk.t4)):
                idx.setdefault(row, j)  # the lowest table index of each row
            self.J = []
            for i in range(n):
                row = (self.A[i], self.B[i], self.C[i], pk.qtag[i])
                assert not pk.qk[i] or row in idx, "lookup row %d is not in the table" % i
                self.J.append(idx[row] if pk.qk[i] else 0)
        self.Ab, self.Bb, self.Cb = (self._blind(k, v) for k, v in zip("ABC", W))
        return {"a_1": commit_coeffs(self.setup, self.Ab), "b_1": commit_coeffs(self.setup, self.Bb),
                "c_1": commit_coeffs(self.setup, self.Cb)}

    def round_1L(self):
        """t = t1 + eta t2 + eta^2 t3 + eta^3 t4, f = t at each lookup row's table row, s = (f, t) sorted by t, split
        alternately into H1, H2"""
        n, pk, eta = self.n, self.pk, self.eta
        e2, e3 = eta * eta % R, pow(eta, 3, R)
        self.Tl = [(x + eta * y + e2 * z + e3 * g) % R for x, y, z, g in zip(*pk.table, pk.t4)]
        self.F = [self.Tl[j] for j in self.J]
        s = [self.Tl[j] for j in sorted(list(range(n)) + self.J)]
        self.H1, self.H2 = s[0::2], s[1::2]
        self.Fb, self.H1b, self.H2b = (self._blind(k, v) for k, v in (("F", self.F), ("H1", self.H1), ("H2", self.H2)))
        return {"f_1": commit_coeffs(self.setup, self.Fb), "h1_1": commit_coeffs(self.setup, self.H1b),
                "h2_1": commit_coeffs(self.setup, self.H2b)}

    def round_2(self):
        """the grand products: the permutation's Z, the shuffle's Z3, the lookup's Z2; each must close"""
        n, pk, be, ga = self.n, self.pk, self.beta, self.gamma
        A, B, C, roots = self.A, self.B, self.C, O.roots_of_unity(n)
        Z = [1]
        for i in range(n):
            num = (A[i] + be * roots[i] + ga) * (B[i] + 2 * be * roots[i] + ga) % R * (C[i] + 3 * be * roots[i] + ga)
            den = (A[i] + be * pk.S1[i] + ga) * (B[i] + be * pk.S2[i] + ga) % R * (C[i] + be * pk.S3[i] + ga)
            Z.append(Z[-1] * num % R * O.inv0(den, R) % R)
        assert Z.pop() == 1, "permutation grand product does not close"
        self.Z, self.Zb = Z, self._blind("Z", Z)
        out = {"z_1": commit_coeffs(self.setup, self.Zb)}
        if "shuffle" in self.blocks:
            th, Z3 = self.theta, [1]
            for i in range(n):
                t = (self.kappa + A[i] + th * B[i] + th * th % R * C[i]) % R
                Z3.append(Z3[-1] * (t if pk.q_in[i] else 1) % R * O.inv0(t if pk.q_out[i] else 1, R) % R)
            assert Z3.pop() == 1, NOT_A_SHUFFLE
            self.Z3, self.Z3c = Z3, self._blind("Z3", Z3)
            out["z3_1"] = commit_coeffs(self.setup, self.Z3c)
        if "lookup" in self.blocks:
            d, e, T, F_, H1, H2 = self.delta, self.epsilon, self.Tl, self.F, self.H1, self.H2
            od, eod = (1 + d) % R, e * (1 + d) % R
            Z2 = [1]
            for i in range(n):
                i1 = (i + 1) % n
                num = od * (e + F_[i]) % R * (eod + T[i] + d * T[i1]) % R
                den = (eod + H1[i] + d * H2[i]) % R * ((eod + H2[i] + d * H1[i1]) % R) % R
                Z2.append(Z2[-1] * num % R * O.inv0(den, R) % R)
            assert Z2.pop() == 1, "lookup grand product does not close"
            self.Z2, self.Z2b = Z2, self._blind("Z2", Z2)
            out["z2_1"] = commit_coeffs(self.setup, self.Z2b)
        return out

    def round_3(self):
        """T = (gate + alpha perm + alpha^2 L0 (Z - 1) + the shuffle's or the lookup's terms) / Z_H on the 4n coset,
        then cut into T1', T2', T3'"""
        n, pk, b = self.n, self.pk, self.blinders
        xs = [self.fft_cofactor * m % R for m in O.roots_of_unity(4 * n)]
        ZH = [(pow(x, n, R) - 1) % R for x in xs]
        ext = self._ext

        def blinded(name, values):  # the blinded polynomial on the coset
            zc = self._zh(name)
            return [(e + poly_eval(zc, x) * zh) % R for e, x, zh in zip(ext(values), xs, ZH)]

        def sh(v):  # X -> wX on the 4x finer domain
            return v[4:] + v[:4]
        A, B, C, Z = blinded("A", self.A), blinded("B", self.B), blinded("C", self.C), blinded("Z", self.Z)
        S1, S2, S3, L0 = ext(pk.S1), ext(pk.S2), ext(pk.S3), ext([1] + [0] * (n - 1))
        al, be, ga = self.alpha, self.beta, self.gamma
        al2, al3 = al * al % R, pow(al, 3, R)
        al4, al5 = al3 * al % R, pow(al, 5, R)
        num = gate([ext(q) for q in (pk.QL, pk.QR, pk.QM, pk.QO, pk.QC)], ext(self.PI),
                   [(e, ext(q)) for e, q in pk.custom], A, B, C, 4)
        Zw = sh(Z)
        for j, x in enumerate(xs):
            a, bb, c = A[j], B[j], C[j]
            p1 = (a + be * x + ga) * (bb + 2 * be * x + ga) % R * (c + 3 * be * x + ga) % R
            p2 = (a + be * S1[j] + ga) * (bb + be * S2[j] + ga) % R * (c + be * S3[j] + ga) % R
            num[j] += al * (p1 * Z[j] - p2 * Zw[j]) + al2 * (Z[j] - 1) * L0[j]
        if "shuffle" in self.blocks:
            Z3, QI, QO, th = blinded("Z3", self.Z3), ext(pk.q_in), ext(pk.q_out), self.theta
            Z3w = sh(Z3)
            for j in range(4 * n):
                K = (self.kappa + A[j] + th * B[j] + th * th % R * C[j] - 1) % R
                num[j] += al3 * (Z3w[j] * (1 + QO[j] * K) - Z3[j] * (1 + QI[j] * K)) + al4 * (Z3[j] - 1) * L0[j]
        if "lookup" in self.blocks:
            eta, d, e = self.eta, self.delta, self.epsilon
            od, eod, e3 = (1 + d) % R, e * (1 + d) % R, pow(eta, 3, R)
            QK, QT, T = ext(pk.qk), ext(pk.qtag), ext(self.Tl)
            Fv, H1, H2, Z2 = (blinded(k, v) for k, v in (("F", self.F), ("H1", self.H1), ("H2", self.H2),
                                                         ("Z2", self.Z2)))
            Tw, H1w, Z2w = sh(T), sh(H1), sh(Z2)
            for j in range(4 * n):
                lk1 = QK[j] * (A[j] + eta * B[j] + eta * eta % R * C[j] - Fv[j]) + e3 * QT[j]
                lk2 = (Z2[j] * od % R * (e + Fv[j]) % R * ((eod + T[j] + d * Tw[j]) % R)
                       - Z2w[j] * ((eod + H1[j] + d * H2[j]) % R) % R * ((eod + H2[j] + d * H1w[j]) % R))
                num[j] += al3 * lk1 + al4 * lk2 + al5 * (Z2[j] - 1) * L0[j]
        T = O.coset_extended_lagrange_to_coeffs([v % R * O.inv0(zh, R) % R for v, zh in zip(num, ZH)],
                                                self.fft_cofactor)
        top = 3 * n + (9 if "next_row" in self.blocks else 6) if any(b) else 3 * n
        assert not any(T[top:]), "deg T >= %d" % top
        self.T = T
        b10, b11 = (b[i] for i in self.layout["T"])
        self.T1b = T[:n] + [b10]
        self.T2b = [(T[n] - b10) % R] + T[n + 1:2 * n] + [b11]
        self.T3b = [(T[2 * n] - b11) % R] + T[2 * n + 1:top]
        return {k: commit_coeffs(self.setup, p) for k, p in (("t_lo_1", self.T1b), ("t_mid_1", self.T2b),
                                                             ("t_hi_1", self.T3b))}

    def round_4(self):
        """the committed polynomials by Horner at zeta or zeta w, the fixed columns by barycentric evaluation"""
        z, pk = self.zeta, self.pk
        zw = z * O.root_of_unity(self.n) % R
        ev = {"a_eval": poly_eval(self.Ab, z), "b_eval": poly_eval(self.Bb, z), "c_eval": poly_eval(self.Cb, z),
              "s1_eval": O.barycentric_eval(pk.S1, z), "s2_eval": O.barycentric_eval(pk.S2, z),
              "z_shifted_eval": poly_eval(self.Zb, zw)}
        if "next_row" in self.blocks:
            ev.update(zip(FIELDS["next_row"]["4"], (poly_eval(p, zw) for p in (self.Ab, self.Bb, self.Cb))))
        if "shuffle" in self.blocks:
            ev.update(qin_eval=O.barycentric_eval(pk.q_in, z), z3_shifted_eval=poly_eval(self.Z3c, zw))
        if "lookup" in self.blocks:
            ev.update(f_eval=poly_eval(self.Fb, z), t_eval=O.barycentric_eval(self.Tl, z),
                      t_shifted_eval=O.barycentric_eval(self.Tl, zw), h2_eval=poly_eval(self.H2b, z),
                      h1_shifted_eval=poly_eval(self.H1b, zw), z2_shifted_eval=poly_eval(self.Z2b, zw))
        self.ev = ev
        return ev

    def round_5(self):
        """W_z = (R + sum_i v^i (P_i - p_i)) / (X - zeta), W_zw = sum_i v^i (P_i - p_i) / (X - zeta w)"""
        pk, n, v = self.pk, self.n, self.v
        P = {k: O.ifft(col) for k, col in (("Ql", pk.QL), ("Qr", pk.QR), ("Qm", pk.QM), ("Qo", pk.QO), ("Qc", pk.QC),
                                           ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
        P.update(custom=[(e, O.ifft(q)) for e, q in pk.custom], A=self.Ab, B=self.Bb, C=self.Cb, Z=self.Zb,
                 T1=self.T1b, T2=self.T2b, T3=self.T3b)
        if "shuffle" in self.blocks:
            P.update(Qin=O.ifft(pk.q_in), Qout=O.ifft(pk.q_out), Z3=self.Z3c)
        if "lookup" in self.blocks:
            P.update(Qk=O.ifft(pk.qk), Qt=O.ifft(pk.qtag), T=O.ifft(self.Tl), F=self.Fb, H1=self.H1b, H2=self.H2b,
                     Z2=self.Z2b)
        ch = {k: getattr(self, k) for k in ("alpha", "beta", "gamma", "zeta", "theta", "kappa", "eta", "delta",
                                            "epsilon") if hasattr(self, k)}
        terms, r0, at_z, at_zw = linearisation(self.blocks, n, ch, self.ev, O.barycentric_eval(self.PI, self.zeta), P)
        num = lincomb(terms + [(p, pow(v, i, R)) for i, (p, _) in enumerate(at_z, 1)])
        num[0] = (num[0] + r0 - sum(pow(v, i, R) * x for i, (_, x) in enumerate(at_z, 1))) % R
        numw = lincomb([(p, pow(v, i, R)) for i, (p, _) in enumerate(at_zw)])
        numw[0] = (numw[0] - sum(pow(v, i, R) * x for i, (_, x) in enumerate(at_zw))) % R
        Wz = divide_linear(num, self.zeta)
        Wzw = divide_linear(numw, self.zeta * O.root_of_unity(n) % R)
        return {"W_z_1": commit_coeffs(self.setup, Wz), "W_zw_1": commit_coeffs(self.setup, Wzw)}


def prove(setup, pk: Preprocessed, A, B, C, public_inputs, blinders=None, fast: bool = False,
          check: bool = True) -> dict:
    """the oracle's proof; ``blinders``: b1..bm for zero-knowledge mode (m = blinder_count(pk)), None for zeros;
    ``fast``: transforms by the C restatement (setup: an oracle.fast.Setup).  The SRS needs n powers without blinders,
    n + 6 with (n + 9 with next-row terms)."""
    if fast:
        with F.c_kernels():
            return Prover(setup, pk, blinders, check).prove(A, B, C, public_inputs)
    return Prover(setup, pk, blinders, check).prove(A, B, C, public_inputs)


# ---- the verifier --------------------------------------------------------------------------------------------------
def verify_proof_trapdoor(group_order: int, vk: dict, proof: dict, public, tau: int) -> bool:
    """the batched verifier with the final pairing equation checked through tau: e(W_z + u W_zw, [tau]_2) ==
    e(zeta W_z + u zeta w W_zw + F - [E] G, G2) holds iff tau (W_z + u W_zw) == zeta W_z + u zeta w W_zw + F - E G.
    vk: G1 points Qm Ql Qr Qo Qc S1 S2 S3, and optionally "custom": [(exponents, [Q_k])] in the prover's order,
    "shuffle": ([q_in], [q_out]), "lookup": ([q_K], [t1], [t2], [t3]) or with ([Q_T], [t4]) after them; None for a
    zero column"""
    n, blocks = group_order, proof_kind(proof)
    ch = challenges(proof)
    zeta, v, u = ch["zeta"], ch["v"], ch["u"]
    w = O.root_of_unity(n)
    ZH = (pow(zeta, n, R) - 1) % R
    pi = sum((-p) * pow(w, i, R) % R * ZH % R * O.inv0(n * (zeta - pow(w, i, R)), R) for i, p in enumerate(public)) % R
    P = dict(vk, custom=vk.get("custom", []), A=proof["a_1"], B=proof["b_1"], C=proof["c_1"], Z=proof["z_1"],
             T1=proof["t_lo_1"], T2=proof["t_mid_1"], T3=proof["t_hi_1"])
    if "shuffle" in blocks:
        P.update(Qin=vk["shuffle"][0], Qout=vk["shuffle"][1], Z3=proof["z3_1"])
    if "lookup" in blocks:
        qk, t1, t2, t3, qt, t4 = tuple(vk["lookup"]) + (None, None) * (len(vk["lookup"]) == 4)
        eta = ch["eta"]
        T = [(p, pow(eta, i, R)) for i, p in enumerate((t1, t2, t3, t4)) if p is not None]
        P.update(Qk=qk, Qt=qt, T=O.ec_lincomb_naive(T), F=proof["f_1"], H1=proof["h1_1"], H2=proof["h2_1"],
                 Z2=proof["z2_1"])
    terms, r0, at_z, at_zw = linearisation(blocks, n, ch, proof, pi, P)
    pts = terms + [(p, pow(v, i, R)) for i, (p, _) in enumerate(at_z, 1)]
    pts += [(p, u * pow(v, i, R)) for i, (p, _) in enumerate(at_zw)]
    E = (-r0 + sum(pow(v, i, R) * x for i, (_, x) in enumerate(at_z, 1))
         + u * sum(pow(v, i, R) * x for i, (_, x) in enumerate(at_zw))) % R
    Fp = O.ec_lincomb_naive([(p, k % R) for p, k in pts if p is not None])
    lhs = O.g1_multiply(O.ec_lincomb_naive([(proof["W_z_1"], 1), (proof["W_zw_1"], u)]), tau)
    rhs = O.ec_lincomb_naive([(proof["W_z_1"], zeta), (proof["W_zw_1"], u * zeta % R * w), (Fp, 1), (O.G1, -E % R)])
    return lhs == rhs
