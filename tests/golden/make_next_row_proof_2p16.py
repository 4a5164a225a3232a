"""Generates tests/golden/proof_next_row_2p16.json: the oracle's proof of a 2^16-row circuit of 16-bit range checks by the
running sum over the next row (plonkathon_b200/synthetic.py ``range_check_circuit``: the four custom terms a(wX)^2,
a a(wX), a^2, a(wX) of the running-sum gate on 16 of every 17 rows), on a structured SRS of n powers with the test tau.
tests/test_next_row.py proves the same circuit on the GPU and compares the bytes.

The prover is tests/next_row_oracle.py over the C restatement of fft / ec_lincomb (oracle/fast.py).  One core, a few
minutes:

    python tests/golden/make_next_row_proof_2p16.py
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
from tests import next_row_oracle as NR  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, BITS, SEED = 16, 16, 16
N_VALUES = ((1 << LOG_N) - 2) // (BITS + 1)
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


c = syn.range_check_circuit(LOG_N, N_VALUES, bits=BITS, seed=SEED)
n = c.group_order
pk = NR.preprocessed(c)
A, B, C = c.wires_values()
log("circuit built: %d values, %d rows" % (N_VALUES, c.n_constraints))
setup = F.Setup(TAU, n)
proof = NR.prove(setup, pk, A, B, C, [], fast=True)
raw = NR.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    custom = [(e, setup.commit(col)) for e, col in c.custom]
assert NR.verify_proof_trapdoor(n, vk, custom, proof, [], TAU)
log("trapdoor check passed")
rec = {"log_n": LOG_N, "bits": BITS, "n_values": N_VALUES, "seed": SEED, "tau": hex(TAU), "srs_powers": n,
       "terms": [list(e) for e, _ in c.custom], "vk_custom": [[list(e), [str(p[0]), str(p[1])]] for e, p in custom],
       "public": [], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "generator": "tests/golden/make_next_row_proof_2p16.py (tests/next_row_oracle.py over oracle/fast.py)",
       "seconds": round(time.time() - t0, 1)}
out = os.path.join(HERE, "proof_next_row_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
