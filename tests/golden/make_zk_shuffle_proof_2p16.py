"""Generates tests/golden/proof_zk_shuffle_2p16.json: the oracle's zero-knowledge proof of the circuit of
proof_shuffle_2p16.json (2^16 rows, four next-row custom gate terms, a shuffle of a quarter of the rows) with 17 fixed
nonzero blinders, on a structured SRS of n + 9 powers with the test tau.  tests/test_zk_shuffle.py proves the same
circuit with the same blinders on the GPU and compares the bytes.

The prover is tests/zk_shuffle_oracle.py over the C restatement of fft / ec_lincomb (oracle/fast.py).  One core, a few
minutes:

    python tests/golden/make_zk_shuffle_proof_2p16.py
"""
import hashlib
import json
import os
import random
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import fast as F  # noqa: E402
from oracle import plonk_oracle as O  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402
from tests import shuffle_oracle as SO  # noqa: E402
from tests import zk_shuffle_oracle as ZS  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, SEED, N_PUBLIC, BLINDER_SEED = 16, 16, 2, 2016
TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


c = syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, custom=TERMS, shuffle=True)
n = c.group_order
pk = SO.preprocessed(c)
A, B, C = c.wires_values()
public = c.public_values()
rng = random.Random(BLINDER_SEED)
blinders = [rng.randrange(1, O.R_MOD) for _ in range(ZS.N_NEXT_ROW_BLINDERS)]
log("circuit built: %d rows, %d in-rows, %d out-rows" % (c.n_constraints, sum(c.shuffle[0]), sum(c.shuffle[1])))
setup = F.Setup(TAU, n + 9)
proof = ZS.prove(setup, pk, A, B, C, public, blinders, fast=True)
raw = SO.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom = [(e, setup.commit(col)) for e, col in c.custom]
    shuffle = tuple(setup.commit(q) for q in c.shuffle)
assert SO.verify_proof_trapdoor(n, vk, custom, shuffle, proof, public, TAU)
log("trapdoor check passed")
rec = {"log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "tau": hex(TAU), "srs_powers": n + 9,
       "terms": [list(e) for e, _ in c.custom], "rows_in": sum(c.shuffle[0]), "blinders": [str(b) for b in blinders],
       "public": [str(x) for x in public], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "generator": "tests/golden/make_zk_shuffle_proof_2p16.py (tests/zk_shuffle_oracle.py over oracle/fast.py)"}
out = os.path.join(HERE, "proof_zk_shuffle_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
