"""TEST INFRASTRUCTURE ONLY -- the oracle prover and trapdoor verifier for lookups over several tables (a table tag).

PlonKup's table tag over tests/lookup_oracle.py, as DESIGN.md fixes it: the tables are concatenated, t4 holds each table
row's id and the fixed selector Q_T the id of the table each lookup row reads (0 elsewhere).  A lookup row matches
(a, b, c, Q_T) against (t1, t2, t3, t4); t gains eta^3 t4; the quotient's alpha^3 term gains alpha^3 eta^3 Q_T and the
linearisation alpha^3 eta^3 [Q_T]; the verifier forms [T] with eta^3 [t4].

``TaggedProver`` reuses ``LookupProver``'s rounds 3 and 5 unchanged: alpha^3 eta^3 Q_T has weight 1 in both the quotient
and the linearisation, exactly like the constant selector QC, so they run with QC + alpha^3 eta^3 Q_T in QC's place
(fft_expand is linear).  The trapdoor check likewise runs ``lookup_oracle.verify_proof_trapdoor`` with
[QC] + alpha^3 eta^3 [Q_T] and [t1] + eta^3 [t4].  With Q_T = t4 = 0 every added term is zero."""
from __future__ import annotations

import contextlib
import dataclasses
from dataclasses import dataclass, field

from oracle import fast as F
from oracle import plonk_oracle as O
from tests import custom_gate_oracle as CG
from tests import lookup_oracle as LK

R = O.R_MOD


@dataclass
class TaggedPreprocessed(LK.LookupPreprocessed):
    qtag: list = field(default_factory=list)  # Q_T: n values, the table id of each lookup row, 0 elsewhere
    t4: list = field(default_factory=list)    # each table row's id, padded to n as the table


class TaggedProver(LK.LookupProver):
    def round_1(self, A, B, C):
        out = CG.CustomProver.round_1(self, A, B, C)
        idx = LK.table_index(self.pk.table + [self.pk.t4])
        self.J = []
        for i in range(self.group_order):
            if self.pk.qk[i]:
                row = (self.A[i], self.B[i], self.C[i], self.pk.qtag[i])
                assert row in idx, "lookup row %d is not in the table" % i
                self.J.append(idx[row])
            else:
                self.J.append(0)
        return out

    def round_lookup(self):
        eta3 = pow(self.eta, 3, R)
        table = self.pk.table
        # t1 + eta^3 t4 in t1's place: LookupProver.round_lookup then builds t = t1 + eta t2 + eta^2 t3 + eta^3 t4
        t1 = [(x + eta3 * g) % R for x, g in zip(table[0], self.pk.t4)]
        with self._pk(table=[t1] + table[1:]):
            return super().round_lookup()

    def round_3(self):
        with self._pk(QC=self._qc_tagged()):
            return super().round_3()

    def round_5(self):
        with self._pk(QC=self._qc_tagged()):
            return super().round_5()

    def _qc_tagged(self):
        """QC + alpha^3 eta^3 Q_T"""
        w = pow(self.alpha, 3, R) * pow(self.eta, 3, R) % R
        return [(x + w * q) % R for x, q in zip(self.pk.QC, self.pk.qtag)]

    @contextlib.contextmanager
    def _pk(self, **changes):
        """self.pk with some fields replaced, for the duration of a ``with``"""
        saved = self.pk
        self.pk = dataclasses.replace(saved, **changes)
        try:
            yield
        finally:
            self.pk = saved


def prove(setup, pk: TaggedPreprocessed, A, B, C, public_inputs, fast: bool = False) -> dict:
    if fast:
        with F.c_kernels():
            return TaggedProver(setup, pk).prove(A, B, C, public_inputs)
    return TaggedProver(setup, pk).prove(A, B, C, public_inputs)


def verify_proof_trapdoor(group_order: int, vk: dict, custom_pts, lookup_pts, proof: dict, public, tau: int) -> bool:
    """the batched verifier of a tagged lookup proof with the final pairing equation checked through tau.
    lookup_pts: ([q_K], [t1], [t2], [t3], [Q_T], [t4]), or the first four for one untagged table; None for the
    identity."""
    qk, t1, t2, t3, *tag = lookup_pts
    if tag:
        qt, t4 = tag
        ch = LK.challenges(proof)
        eta3 = pow(ch["eta"], 3, R)
        a3e3 = pow(ch["alpha"], 3, R) * eta3 % R
        vk = dict(vk, Qc=O.ec_lincomb_naive([(p, k) for p, k in ((vk["Qc"], 1), (qt, a3e3)) if p is not None]))
        t1 = O.ec_lincomb_naive([(p, k) for p, k in ((t1, 1), (t4, eta3)) if p is not None])
    return LK.verify_proof_trapdoor(group_order, vk, custom_pts, (qk, t1, t2, t3), proof, public, tau)


def preprocessed(c, S=None) -> TaggedPreprocessed:
    """TaggedPreprocessed of a plonkathon_b200.synthetic.ArrayCircuit with lookups over several tables (``lookups=``)
    or one table (``lookup=``; zero Q_T and t4)"""
    from plonkathon_b200.lookup import check_lookups, padded_table
    n = c.group_order
    lookups = c.lookups or [c.lookup]
    base = LK.preprocessed(dataclasses.replace(c, lookup=lookups[0]), S)
    qk, qtag, cols, _ = check_lookups(lookups, n)
    *table, t4 = padded_table(cols, n)
    return TaggedPreprocessed(**{f.name: getattr(base, f.name) for f in dataclasses.fields(base)} |
                              {"qk": qk, "table": table}, qtag=qtag, t4=t4)
