"""Generates tests/golden/proof_lookup_2p16.json: the oracle's lookup proof of a 2^16-gate synthetic circuit of the
bench family (two public inputs) with lookup rows into a range table of 2^15 rows (t1 = 0 .. 2^15 - 1, t2 = t3 = 0),
structured SRS with the test tau.  tests/test_lookup.py proves the same circuit on the GPU and compares the bytes.

The prover is tests/lookup_oracle.py over the C restatement of fft / ec_lincomb (oracle/fast.py).  One core, a few
minutes:

    python tests/golden/make_lookup_proof_2p16.py
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
from tests import lookup_oracle as LK  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, SEED, N_PUBLIC, TABLE_ROWS = 16, 16, 2, 1 << 15
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


table = [list(range(TABLE_ROWS)), [0] * TABLE_ROWS, [0] * TABLE_ROWS]
c = syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, lookup=table)
n = c.group_order
pk = LK.preprocessed(c)
A, B, C = c.wires_values()
log("circuit built: %d lookup rows" % sum(c.lookup[0]))
setup = F.Setup(TAU, n)
proof = LK.prove(setup, pk, A, B, C, c.public_values(), fast=True)
raw = LK.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    lk = (setup.commit(pk.qk), setup.commit(pk.table[0]), None, None)
assert LK.verify_proof_trapdoor(n, vk, [], lk, proof, c.public_values(), TAU)
log("trapdoor check passed")
rec = {"log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "tau": hex(TAU), "table": "range", "table_rows": TABLE_ROWS,
       "public": [str(x) for x in c.public_values()], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "vk_lookup": [None if p is None else [str(p[0]), str(p[1])] for p in lk],
       "generator": "tests/golden/make_lookup_proof_2p16.py (tests/lookup_oracle.py over oracle/fast.py)",
       "seconds": round(time.time() - t0, 1)}
out = os.path.join(HERE, "proof_lookup_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
