"""Generates tests/golden/proof_zk_lookup_2p16.json: the oracle's zero-knowledge lookup proof of the 2^16-gate circuit of
tests/golden/proof_tagged_lookup_2p16.json (bench family, two public inputs, lookups over an 8-bit range table, a 4-bit
XOR table and a 4-bit AND table) with 21 fixed nonzero blinders, on a structured SRS of n + 6 powers with the test tau.
tests/test_zk_lookup.py proves the same circuit with the same blinders on the GPU and compares the bytes.

The prover is tests/zk_lookup_oracle.py over the C restatement of fft / ec_lincomb (oracle/fast.py).  One core, a few
minutes:

    python tests/golden/make_zk_lookup_proof_2p16.py
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
from tests import lookup_oracle as LK  # noqa: E402
from tests import tagged_lookup_oracle as TL  # noqa: E402
from tests import zk_lookup_oracle as ZL  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, SEED, N_PUBLIC, BLINDER_SEED = 16, 16, 2, 2022086
t0 = time.time()


def log(msg):
    print("[%7.1f s] %s" % (time.time() - t0, msg), flush=True)


def op_table(bits, op):
    rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(c) for c in zip(*rows)]


tables = [[list(range(256)), [0] * 256, [0] * 256], op_table(4, lambda x, y: x ^ y), op_table(4, lambda x, y: x & y)]
c = syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, lookups=tables)
n = c.group_order
pk = TL.preprocessed(c)
A, B, C = c.wires_values()
rng = random.Random(BLINDER_SEED)
blinders = [rng.randrange(1, O.R_MOD) for _ in range(ZL.N_BLINDERS)]
log("circuit built: lookup rows per table %s" % [sum(q) for q, _ in c.lookups])
setup = F.Setup(TAU, n + 6)
proof = ZL.prove(setup, pk, A, B, C, c.public_values(), blinders, fast=True)
raw = LK.proof_bytes(proof)
log("proof done")
with F.c_kernels():
    vk = {name: setup.commit(col) for name, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                                     ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
    lk = tuple(None if not any(col) else setup.commit(col) for col in [pk.qk] + pk.table + [pk.qtag, pk.t4])
assert TL.verify_proof_trapdoor(n, vk, [], lk, proof, c.public_values(), TAU)
log("trapdoor check passed")
rec = {"log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "tau": hex(TAU), "srs_powers": n + 6,
       "tables": ["range 8-bit (v, 0, 0)", "xor 4-bit", "and 4-bit"], "table_rows": [len(t[0]) for t in tables],
       "blinder_seed": BLINDER_SEED, "blinders": [str(b) for b in blinders],
       "public": [str(x) for x in c.public_values()], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
       "generator": "tests/golden/make_zk_lookup_proof_2p16.py (tests/zk_lookup_oracle.py over oracle/fast.py)",
       "seconds": round(time.time() - t0, 1)}
out = os.path.join(HERE, "proof_zk_lookup_2p16.json")
json.dump(rec, open(out, "w"), indent=1)
log("wrote " + out + " sha256 " + rec["sha256"])
