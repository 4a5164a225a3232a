"""Generates tests/golden/proof_zk_2p16.json: the oracle's zero-knowledge proof of a 2^16-gate synthetic circuit of the
bench family (two public inputs), structured SRS of n + 6 powers with the test tau, and eleven fixed non-zero blinders
drawn from a seeded generator and stored in the fixture.  tests/test_zk.py proves the same circuit on the GPU with the
same blinders and compares the bytes.

The prover is tests/zk_oracle.py (plonk_oracle's rounds with the blinding) over the C restatement of fft / ec_lincomb
(oracle/fast.py).  One core, a few minutes:

    python tests/golden/make_zk_proof_2p16.py
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
from tests import zk_oracle as ZK  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, SEED, N_PUBLIC, BLINDER_SEED = 16, 16, 2, 20261015
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


c = syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC)
n = c.group_order
S = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
pk = O.Preprocessed(n, c.QM, c.QL, c.QR, c.QO, c.QC, *S)
A, B, C = c.wires_values()
rng = random.Random(BLINDER_SEED)
blinders = [rng.randrange(1, O.R_MOD) for _ in range(ZK.N_BLINDERS)]
log("circuit built")
setup = F.Setup(TAU, n + 6)
log("SRS generated")
proof = ZK.prove(setup, pk, A, B, C, c.public_values(), blinders, fast=True)
raw = O.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", S[0]), ("S2", S[1]), ("S3", S[2]))}
log("verification key done")
assert O.verify_proof_trapdoor(n, vk, O.proof_from_bytes(raw), c.public_values(), TAU)
rec = {"log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "tau": hex(TAU), "srs_powers": n + 6,
       "blinder_seed": BLINDER_SEED, "blinders": [str(b) for b in blinders],
       "public": [str(x) for x in c.public_values()], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "vk": {k: [str(v[0]), str(v[1])] for k, v in vk.items()},
       "generator": "tests/golden/make_zk_proof_2p16.py (tests/zk_oracle.py over oracle/fast.py)",
       "seconds": round(time.time() - t0, 1)}
out = os.path.join(HERE, "proof_zk_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
