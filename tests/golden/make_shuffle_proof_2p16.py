"""Generates tests/golden/proof_shuffle_2p16.json: the oracle's proof of a 2^16-row synthetic circuit with four next-row
custom gate terms and a shuffle (plonkathon_b200/synthetic.py ``build_circuit(..., shuffle=True)``: a quarter of the
rows are out-rows holding the (a, b, c) of another quarter, the in-rows, in a random order), on a structured SRS of n
powers with the test tau.  tests/test_shuffle.py proves the same circuit on the GPU and compares the bytes.

The prover is tests/shuffle_oracle.py over the C restatement of fft / ec_lincomb (oracle/fast.py).  One core, a few
minutes:

    python tests/golden/make_shuffle_proof_2p16.py
"""
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import fast as F  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402
from tests import shuffle_oracle as SO  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, SEED, N_PUBLIC = 16, 16, 2
TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


c = syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, custom=TERMS, shuffle=True)
n = c.group_order
pk = SO.preprocessed(c)
A, B, C = c.wires_values()
public = c.public_values()
log("circuit built: %d rows, %d in-rows, %d out-rows" % (c.n_constraints, sum(c.shuffle[0]), sum(c.shuffle[1])))
setup = F.Setup(TAU, n)
proof = SO.prove(setup, pk, A, B, C, public, fast=True)
raw = SO.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom = [(e, setup.commit(col)) for e, col in c.custom]
    shuffle = tuple(setup.commit(q) for q in c.shuffle)
assert SO.verify_proof_trapdoor(n, vk, custom, shuffle, proof, public, TAU)
log("trapdoor check passed")
rec = {"log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "tau": hex(TAU), "srs_powers": n,
       "terms": [list(e) for e, _ in c.custom], "rows_in": sum(c.shuffle[0]),
       "vk_shuffle": [[str(p[0]), str(p[1])] for p in shuffle], "public": [str(x) for x in public],
       "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "generator": "tests/golden/make_shuffle_proof_2p16.py (tests/shuffle_oracle.py over oracle/fast.py)",
       "seconds": round(time.time() - t0, 1)}
out = os.path.join(HERE, "proof_shuffle_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
