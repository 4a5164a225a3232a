#!/usr/bin/env python
"""Write tests/golden/solve_programs.json by running the reference compiler (``Program.wires``,
``common_preprocessed_input`` and ``fill_variable_assignments``, compiler/program.py) on the factorization, mini-Poseidon
and prover_test programs of its test.py, over the restated third-party layer in ``oracle/shims``.

Only runnable where the reference tree is available (REF below); the fixture it writes is what
tests/test_solve.py reads.  Per program: the cell ids (``program.wires()`` with variable names numbered in order of first
appearance, None as -1), the gate selectors QL QR QM QO QC, the starting assignments test.py passes (by id), and
the SHA-256 of each column A, B, C of ``fill_variable_assignments``' output (32-byte little-endian values, None as 0).
Values are written as signed decimal strings: x as x - r when that is shorter."""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get("PLONKATHON_REF", "/root/reference")
sys.path.insert(0, os.path.join(ROOT, "oracle", "shims"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)
os.chdir(REF)

from compiler.program import Program  # noqa: E402  reference compiler
from test.mini_poseidon import rc, mds  # noqa: E402  reference

R = 21888242871839275222246405745257275088548364400416034343698204186575808495617


def output_proof_lang():
    """the mini-Poseidon program of test.py:216-259 (as make_golden.py builds it)"""
    o = ["L0 public", "M0 public", "M64 public", "R0 <== 0"]
    for i in range(64):
        for j, pos in enumerate(("L", "M", "R")):
            f = {"x": i, "r": rc[i][j], "p": pos}
            if i < 4 or i >= 60 or pos == "L":
                o.append("{p}adj{x} <== {p}{x} + {r}".format(**f))
                o.append("{p}sq{x} <== {p}adj{x} * {p}adj{x}".format(**f))
                o.append("{p}qd{x} <== {p}sq{x} * {p}sq{x}".format(**f))
                o.append("{p}qn{x} <== {p}qd{x} * {p}adj{x}".format(**f))
            else:
                o.append("{p}qn{x} <== {p}{x} + {r}".format(**f))
        for j, pos in enumerate(("L", "M", "R")):
            o.append("{p}suma{x} <== Lqn{x} * {m}".format(x=i, p=pos, m=mds[j]))
            o.append("{p}sumb{x} <== {p}suma{x} + Mqn{x} * {m}".format(x=i, p=pos, m=mds[j + 1]))
            o.append("{p}{xp1} <== {p}sumb{x} + Rqn{x} * {m}".format(
                x=i, xp1=i + 1, p=pos, m=mds[j + 2]))
    return "\n".join(o)


def signed(x):
    x = int(x) % R
    return str(x - R if x > R // 2 else x)


def digest(ints):
    return hashlib.sha256(b"".join((int(x) % R).to_bytes(32, "little") for x in ints)).hexdigest()


def entry(program, start):
    wires = program.wires()
    ids = {}
    for w in wires:
        for name in (w.L, w.R, w.O):
            if name is not None and name not in ids:
                ids[name] = len(ids)
    cell = lambda name: -1 if name is None else ids[name]  # noqa: E731
    pk = program.common_preprocessed_input()
    filled = program.fill_variable_assignments(dict(start))
    filled[None] = 0
    return {
        "n": program.group_order,
        "n_constraints": len(wires),
        "wire_L": [cell(w.L) for w in wires],
        "wire_R": [cell(w.R) for w in wires],
        "wire_O": [cell(w.O) for w in wires],
        "selectors": {k: [signed(x.n) for x in getattr(pk, k).values] for k in ("QL", "QR", "QM", "QO", "QC")},
        "inputs": {str(ids[k]): signed(v) for k, v in start.items() if k in ids},
        "columns_sha256": {col: digest([filled[getattr(w, wire)] for w in wires])
                           for col, wire in (("A", "L"), ("B", "R"), ("C", "O"))},
    }


out = {
    "prover_test": entry(Program(["e public", "c <== a * b", "e <== c * d"], 8),
                         {"a": 3, "b": 4, "c": 12, "d": 5, "e": 60}),
    "factorization": entry(Program.from_str(
        """n public
        pb0 === pb0 * pb0
        pb1 === pb1 * pb1
        pb2 === pb2 * pb2
        pb3 === pb3 * pb3
        qb0 === qb0 * qb0
        qb1 === qb1 * qb1
        qb2 === qb2 * qb2
        qb3 === qb3 * qb3
        pb01 <== pb0 + 2 * pb1
        pb012 <== pb01 + 4 * pb2
        p <== pb012 + 8 * pb3
        qb01 <== qb0 + 2 * qb1
        qb012 <== qb01 + 4 * qb2
        q <== qb012 + 8 * qb3
        n <== p * q""", 16), {"pb3": 1, "pb2": 1, "pb1": 0, "pb0": 1, "qb3": 0, "qb2": 1, "qb1": 1, "qb0": 1}),
    "poseidon": entry(Program.from_str(output_proof_lang(), 1024), {"L0": 1, "M0": 2}),
}
with open(os.path.join(HERE, "solve_programs.json"), "w") as f:
    json.dump(out, f, separators=(",", ":"))
print({k: (v["n_constraints"], v["columns_sha256"]["C"][:12]) for k, v in out.items()})
