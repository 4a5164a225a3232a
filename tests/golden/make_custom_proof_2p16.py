"""Generates tests/golden/proof_custom_2p16.json: the oracle's proof of a 2^16-gate synthetic circuit with all four
custom gate terms of tests/test_custom_gates.py (x^2, z^3, x^2 y, x y z) and two public inputs, structured SRS with the
test tau.  tests/test_custom_gates.py proves the same circuit on the GPU and compares the bytes.

The prover is tests/custom_gate_oracle.py (plonk_oracle's rounds plus the custom terms) over the C restatement of fft /
ec_lincomb (oracle/fast.py).  One core, a few minutes:

    python tests/golden/make_custom_proof_2p16.py
"""
import hashlib
import json
import os
import sys
import time

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import fast as F  # noqa: E402
from oracle import plonk_oracle as O  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402
from tests import custom_gate_oracle as CG  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
TERMS = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]
LOG_N, SEED, N_PUBLIC = 16, 16, 2
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


c = syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, custom=TERMS)
n = c.group_order
pk = CG.preprocessed(c)
A, B, C = c.wires_values()
log("circuit built")
setup = F.Setup(TAU, n)
log("SRS generated")
proof = CG.prove(setup, pk, A, B, C, c.public_values(), fast=True)
raw = O.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom_pts = [(e, setup.commit(col)) for e, col in c.custom]
log("verification key done")
assert CG.verify_proof_trapdoor(n, vk, custom_pts, O.proof_from_bytes(raw), c.public_values(), TAU)
rec = {"log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "terms": [list(e) for e in TERMS], "tau": hex(TAU),
       "public": [str(x) for x in c.public_values()], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "vk": {k: [str(v[0]), str(v[1])] for k, v in vk.items()},
       "vk_custom": [[list(e), [str(p[0]), str(p[1])]] for e, p in custom_pts],
       "generator": "tests/golden/make_custom_proof_2p16.py (tests/custom_gate_oracle.py over oracle/fast.py)",
       "seconds": round(time.time() - t0, 1)}
out = os.path.join(HERE, "proof_custom_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
