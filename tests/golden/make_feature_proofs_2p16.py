"""Golden 2^16-gate proofs of each proof kind by the oracle (tests/extended_oracle.py over the C restatement of fft /
ec_lincomb, oracle/fast.py), checked by its trapdoor verifier before they are written:

    python tests/golden/make_feature_proofs_2p16.py --kind K

with K one of custom, zk, next_row, shuffle, zk_shuffle, lookup, tagged_lookup, zk_lookup, writes
tests/golden/proof_<K>_2p16.json.  One core, a few minutes per kind; the kinds can run in parallel."""
import argparse
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
from tests import extended_oracle as XO  # noqa: E402

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N, SEED, N_PUBLIC = 16, 16, 2
NEXT_TERMS = [(0, 0, 0, 1, 0, 0), (1, 0, 0, 1, 0, 0), (0, 0, 0, 0, 2, 1), (0, 1, 1, 0, 0, 1)]
BITS = 16  # next_row: a running-sum range check of 16-bit values
N_VALUES = ((1 << LOG_N) - 2) // (BITS + 1)


def op_table(bits, op):
    rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(c) for c in zip(*rows)]


RANGE_15 = [list(range(1 << 15)), [0] * (1 << 15), [0] * (1 << 15)]
TABLES = [[list(range(256)), [0] * 256, [0] * 256], op_table(4, lambda x, y: x ^ y), op_table(4, lambda x, y: x & y)]
TABLE_NAMES = ["range 8-bit (v, 0, 0)", "xor 4-bit", "and 4-bit"]

# kind -> (the circuit, blinder seed or None, extra SRS powers, the record's keys in order)
KINDS = {
    "custom": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC,
                                         custom=[(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]), None, 0,
               "log_n seed n_public terms tau public sha256 proof_hex vk vk_custom generator seconds"),
    "zk": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC), 20261015, 6,
           "log_n seed n_public tau srs_powers blinder_seed blinders public sha256 proof_hex vk generator seconds"),
    "next_row": (lambda: syn.range_check_circuit(LOG_N, N_VALUES, bits=BITS, seed=SEED), None, 0,
                 "log_n bits n_values seed tau srs_powers terms vk_custom public sha256 proof_hex generator seconds"),
    "shuffle": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, custom=NEXT_TERMS, shuffle=True),
                None, 0, "log_n seed n_public tau srs_powers terms rows_in vk_shuffle public sha256 proof_hex "
                "generator seconds"),
    "zk_shuffle": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, custom=NEXT_TERMS, shuffle=True),
                   2016, 9, "log_n seed n_public tau srs_powers terms rows_in blinders public sha256 proof_hex "
                   "generator"),
    "lookup": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, lookup=RANGE_15), None, 0,
               "log_n seed n_public tau table table_rows public sha256 proof_hex vk_lookup generator seconds"),
    "tagged_lookup": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, lookups=TABLES), None, 0,
                      "log_n seed n_public tau tables table_rows public sha256 proof_hex vk_lookup generator seconds"),
    "zk_lookup": (lambda: syn.build_circuit(LOG_N, seed=SEED, n_public=N_PUBLIC, lookups=TABLES), 2022086, 6,
                  "log_n seed n_public tau srs_powers tables table_rows blinder_seed blinders public sha256 proof_hex "
                  "generator seconds"),
}


def pt(p):
    return None if p is None else [str(p[0]), str(p[1])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--kind", required=True, choices=sorted(KINDS))
    kind = ap.parse_args().kind
    make, blinder_seed, extra, keys = KINDS[kind]
    t0 = time.time()
    c = make()
    n = c.group_order
    pk = XO.preprocessed(c)
    A, B, C = c.wires_values()
    public = c.public_values()
    blinders = None
    if blinder_seed is not None:
        rng = random.Random(blinder_seed)
        blinders = [rng.randrange(1, O.R_MOD) for _ in range(XO.blinder_count(pk))]
    setup = F.Setup(TAU, n + extra)
    proof = XO.prove(setup, pk, A, B, C, public, blinders, fast=True)
    raw = XO.proof_bytes(proof)
    print("[%7.1f s] proof done" % (time.time() - t0), flush=True)

    def commit(col):
        return setup.commit(col) if any(col) else None  # a zero column commits to the identity
    with F.c_kernels():
        vk = {k: commit(col) for k, col in (("Qm", c.QM), ("Ql", c.QL), ("Qr", c.QR), ("Qo", c.QO), ("Qc", c.QC),
                                            ("S1", pk.S1), ("S2", pk.S2), ("S3", pk.S3))}
        custom = [(e, commit(col)) for e, col in c.custom]
        shuffle = tuple(commit(q) for q in c.shuffle)
        lookup = ()
        if pk.qk is not None:
            lookup = tuple(commit(col) for col in [pk.qk] + pk.table + ([pk.qtag, pk.t4] if c.lookups else []))
    full = dict(vk, custom=custom, shuffle=shuffle, lookup=lookup)
    assert XO.verify_proof_trapdoor(n, full, XO.proof_from_bytes(raw), public, TAU)
    print("[%7.1f s] trapdoor check passed" % (time.time() - t0), flush=True)
    tables = TABLES if c.lookups else [RANGE_15]
    values = {
        "log_n": LOG_N, "seed": SEED, "n_public": N_PUBLIC, "bits": BITS, "n_values": N_VALUES, "tau": hex(TAU),
        "srs_powers": n + extra, "terms": [list(e) for e, _ in c.custom],
        "rows_in": sum(c.shuffle[0]) if c.shuffle else 0,
        "table": "range", "tables": TABLE_NAMES, "table_rows": [len(t[0]) for t in tables] if c.lookups else 1 << 15,
        "blinder_seed": blinder_seed, "blinders": [str(b) for b in blinders or ()],
        "public": [str(x) for x in public], "sha256": hashlib.sha256(raw).hexdigest(), "proof_hex": raw.hex(),
        "vk": {k: pt(p) for k, p in vk.items()}, "vk_custom": [[list(e), pt(p)] for e, p in custom],
        "vk_shuffle": [pt(p) for p in shuffle], "vk_lookup": [pt(p) for p in lookup],
        "generator": "tests/golden/make_feature_proofs_2p16.py --kind %s (tests/extended_oracle.py over oracle/fast.py)"
                     % kind,
        "seconds": round(time.time() - t0, 1)}
    out = os.path.join(HERE, "proof_%s_2p16.json" % kind)
    json.dump({k: values[k] for k in keys.split()}, open(out, "w"), indent=1)
    print("wrote %s sha256 %s" % (out, values["sha256"]))


if __name__ == "__main__":
    main()
