"""CPU: the proof layout is one table in C++ (csrc/proof_layout.cuh, exported by csrc/host_selftest.cpp) and one in
Python (plonkathon_b200/transcript.py).  The two must agree field by field, and each proof kind's filtered table must
give the field order and byte count stated here and by the oracle (tests/extended_oracle.py) independently."""
import ctypes
import os
import subprocess

import pytest

from oracle import plonk_oracle as O
from plonkathon_b200 import transcript as T
from tests import extended_oracle as XO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
BLOCKS = {0: T.PLAIN, 1: T.NEXT_ROW, 2: T.SHUFFLE, 4: T.LOOKUP}  # the C++ block flags


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "build", "host_selftest_layout.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    L = ctypes.CDLL(out)
    L.hs_proof_field.restype = ctypes.c_char_p
    L.hs_proof_challenge.restype = ctypes.c_char_p
    return L


def test_cpp_table_is_python_table(lib):
    ints = [ctypes.c_int() for _ in range(3)]
    fields, k = [], 0
    while (label := lib.hs_proof_field(k, *[ctypes.byref(x) for x in ints])) is not None:
        is_point, step, block = (x.value for x in ints)
        fields.append((label.decode(), "point" if is_point else "scalar", T.STEPS[step], BLOCKS[block]))
        k += 1
    assert tuple(fields) == T.FIELDS
    challenges, k = [], 0
    while (label := lib.hs_proof_challenge(k, *[ctypes.byref(x) for x in ints[:2]])) is not None:
        challenges.append((label.decode(), T.STEPS[ints[0].value], BLOCKS[ints[1].value]))
        k += 1
    assert tuple(challenges) == T.CHALLENGES


NEXT_ROW = ("a_shifted_eval", "b_shifted_eval", "c_shifted_eval")
SHUFFLE = ("z3_1", "qin_eval", "z3_shifted_eval")
LOOKUP = ("f_1", "h1_1", "h2_1", "z2_1", "f_eval", "t_eval", "t_shifted_eval", "h2_eval", "h1_shifted_eval",
          "z2_shifted_eval")


@pytest.mark.parametrize("kind, extension, size", [
    ({}, (), 768),
    ({"next_row": True}, NEXT_ROW, 864),
    ({"shuffle": True}, SHUFFLE, 896),
    ({"next_row": True, "shuffle": True}, NEXT_ROW + SHUFFLE, 992),
    ({"lookup": True}, LOOKUP, 1216),
])
def test_kinds_match_the_oracles(kind, extension, size):
    assert T.proof_fields(**kind) == tuple(O.PROOF_FIELDS) + tuple(extension)
    assert T.proof_bytes(**kind) == size
    assert XO.proof_fields(tuple(kind)) == T.proof_fields(**kind)
