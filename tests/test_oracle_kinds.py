"""CPU: the oracle (tests/extended_oracle.py) proves every record of tests/golden/oracle_kinds.json again with the same
bytes, compared through their SHA-256.  The records cover every proof kind at n = 16 and 64, zero-knowledge kinds
with zero and random blinders (make_oracle_kinds.py lists them), so a change to the oracle's code that moves one proof
byte fails here.  Without custom terms, shuffle, lookups or blinders the oracle gives the bytes of the pinned plain
oracle."""
import hashlib
import json

import pytest

from oracle import fast as F
from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from tests import extended_oracle as XO
from tests.golden.make_oracle_kinds import PATH, TAU, prove_case
from tests.golden_io import ints, load_circuit


def _records():
    return json.load(open(PATH))["records"]


def _id(rec):
    return "%s-%d-%d-%s" % (rec["kind"], rec["log_n"], rec["seed"], rec["blinders"] or "plain")


@pytest.mark.parametrize("rec", _records(), ids=_id)
def test_oracle_reproduces_the_pinned_proof(rec):
    raw = prove_case(rec)
    assert (len(raw), hashlib.sha256(raw).hexdigest()) == (rec["bytes"], rec["sha256"])


@pytest.mark.parametrize("name", ["prover_test", "factorization", "poseidon", "synthetic_256"])
def test_no_blocks_and_no_blinders_give_the_pinned_oracle_proof(name):
    """the oracle of a circuit without custom terms, shuffle or lookups equals oracle/plonk_oracle.py's prover byte for
    byte: on the circuits of tests/golden/circuits.json that have a witness, and on a synthetic one at n = 256"""
    if name == "synthetic_256":
        c = syn.build_circuit(8, seed=5, n_public=3)
        pk, (A, B, C), public = XO.preprocessed(c), c.wires_values(), c.public_values()
    else:
        entry, arr = load_circuit(name)
        pk = XO.Preprocessed(entry["n"], *[arr[k] for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")])
        A, B, C, public = arr["A"], arr["B"], arr["C"], ints(entry["public"])
    setup = F.Setup(TAU, pk.group_order)
    with F.c_kernels():
        plain = O.Prover(setup, pk).prove(A, B, C, public)
        assert XO.proof_bytes(XO.Prover(setup, pk).prove(A, B, C, public)) == O.proof_bytes(plain)
