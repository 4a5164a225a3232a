"""Writes tests/golden/oracle_kinds.json: the SHA-256 of oracle proofs of every proof kind at small sizes, with the
inputs that make them again (kind, log_n, seed, n_public, terms, tables by name, blinders).  tests/test_oracle_kinds.py
proves each record again and compares, so the fixture pins the oracle's bytes across changes to its code.

The kinds: same-row and next-row custom terms; zero knowledge plain, with custom terms and with next-row terms; shuffle
and zero-knowledge shuffle with no terms, same-row terms and next-row terms; one-table lookups over a range, a
duplicate-row and an XOR table, each with and without a custom term; tagged lookups over two and three tables;
zero-knowledge lookups over one, two and three tables.  Zero-knowledge kinds come with zero blinders and with random
ones drawn from the record's seed.  n = 16 and 64, and some at n = 256.  About 15 s in all on one core.

    python tests/golden/make_oracle_kinds.py
"""
import hashlib
import json
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import fast as F  # noqa: E402
from oracle import plonk_oracle as O  # noqa: E402
from plonkathon_b200 import synthetic as syn  # noqa: E402
from tests import extended_oracle as XO  # noqa: E402
from tests.golden_io import GOLDEN  # noqa: E402

PATH = os.path.join(GOLDEN, "oracle_kinds.json")
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
SAME = [[2, 0, 0], [1, 1, 1]]
NEXT = [[0, 0, 0, 1, 0, 0], [1, 0, 0, 1, 0, 0], [0, 0, 0, 0, 2, 1], [0, 1, 1, 0, 0, 1]]


def table(name):
    """"range<k>": (v, 0, 0) for v < k; "xor<b>", "and<b>": (x, y, x op y) for b-bit x, y; "dup": rows 0 and 2, 1 and
    4 equal"""
    if name == "dup":
        rows = [(11, 12, 13), (21, 22, 23), (11, 12, 13), (31, 32, 33), (21, 22, 23), (41, 42, 43)]
    elif name.startswith("range"):
        rows = [(v, 0, 0) for v in range(int(name[5:]))]
    else:
        op, bits = (lambda x, y: x ^ y) if name.startswith("xor") else (lambda x, y: x & y), int(name[3:])
        rows = [(x, y, op(x, y)) for x in range(1 << bits) for y in range(1 << bits)]
    return [list(c) for c in zip(*rows)]


def circuit(rec):
    kw = {"shuffle": True} if rec["kind"] == "shuffle" else {}
    if rec.get("tables"):
        tables = [table(t) for t in rec["tables"]]
        kw.update(lookups=tables) if rec.get("tagged") else kw.update(lookup=tables[0])
    return syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                             custom=[tuple(e) for e in rec["terms"]], **kw)


def prove_case(rec) -> bytes:
    c = circuit(rec)
    pk = XO.preprocessed(c)
    bl = None
    if rec["blinders"] == "zero":
        bl = [0] * XO.blinder_count(pk)
    elif rec["blinders"] == "random":
        rng = random.Random(rec["seed"])
        bl = [rng.randrange(1, O.R_MOD) for _ in range(XO.blinder_count(pk))]
    setup = F.Setup(TAU, c.group_order + 9)
    return XO.proof_bytes(XO.prove(setup, pk, *c.wires_values(), c.public_values(), blinders=bl, fast=True))


def pinned(kind, log_n, terms=(), n_tables=None):
    """the first record without blinders of that kind, size and terms (and number of tables)"""
    for rec in json.load(open(PATH))["records"]:
        if ((rec["kind"], rec["log_n"], rec["terms"], rec["blinders"]) == (kind, log_n, [list(e) for e in terms], None)
                and n_tables in (None, len(rec.get("tables", ())))):
            return rec
    raise KeyError((kind, log_n, terms, n_tables))


def specs():
    out = []
    for log_n in (4, 6):
        n = 1 << log_n
        bits = 1 if n <= 16 else 2
        tagged = ["range%d" % max(2, n // 8), "xor%d" % bits, "and%d" % bits]
        out += [dict(kind="custom", log_n=log_n, terms=SAME), dict(kind="next_row", log_n=log_n, terms=NEXT)]
        out += [dict(kind="zk", log_n=log_n, terms=terms, blind=True) for terms in ([], SAME, NEXT)]
        out += [dict(kind="shuffle", log_n=log_n, terms=terms, blind=blind)
                for terms in ([], SAME, NEXT) for blind in (False, True)]
        out += [dict(kind="lookup", log_n=log_n, terms=terms, tables=[t])
                for t in ("range%d" % (n // 2), "dup") for terms in ([], [[2, 0, 0]])]
        out += [dict(kind="lookup", log_n=log_n, terms=[], tables=tagged[3 - k:], tagged=True) for k in (2, 3)]
        out += [dict(kind="lookup", log_n=log_n, terms=[], tables=tagged[3 - k:], tagged=k > 1, blind=True)
                for k in (1, 2, 3)]
    out += [dict(kind="lookup", log_n=8, terms=terms, tables=["xor4"]) for terms in ([], [[2, 0, 0]])]
    out += [dict(kind="shuffle", log_n=8, terms=terms) for terms in ([], SAME, NEXT)]
    out.append(dict(kind="lookup", log_n=8, terms=[], tables=["range128"]))
    out += [dict(kind="lookup", log_n=8, terms=[], tables=["range32", "xor2", "and2"][3 - k:], tagged=True)
            for k in (2, 3)]
    return out


def records():
    out = []
    for k, spec in enumerate(specs()):
        blind = spec.pop("blind", False)
        seed = 1000 + k
        while True:  # the first seed whose circuit uses every term, table and the shuffle
            c = circuit(dict(spec, seed=seed, n_public=2))
            if (all(any(col) for _, col in c.custom) and (not c.shuffle or any(c.shuffle[0]))
                    and all(any(q) for q, _ in c.lookups or ([c.lookup] if c.lookup else []))):
                break
            seed += 100
        base = dict(spec, seed=seed, n_public=2, blinders=None)
        out += [dict(base, blinders="zero"), dict(base, blinders="random")] if blind else [base]
    return out


def main():
    recs = records()
    for rec in recs:
        raw = prove_case(rec)
        rec.update(bytes=len(raw), sha256=hashlib.sha256(raw).hexdigest())
    with open(PATH, "w") as f:  # one record per line
        f.write('{"generator": "tests/golden/make_oracle_kinds.py", "tau": "%s", "records": [\n' % hex(TAU))
        f.write(",\n".join(json.dumps(r) for r in recs) + "\n]}\n")


if __name__ == "__main__":
    main()
