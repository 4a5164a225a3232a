"""CPU: the copy-constraint permutation's label body (csrc/permutation.cuh), run by csrc/host_selftest.cpp over keys
sorted on the CPU, against synthetic.permutation_polys -- and through it against the reference compiler's digests --
plus the input checks of wiring.permutation_arrays, which refuse bad wirings before the library is called."""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest

from plonkathon_b200 import synthetic as syn
from plonkathon_b200 import wiring
from tests.golden_io import digest, load_json

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
R = syn.R
MAX_ID = (1 << 32) - 2


@pytest.fixture(scope="module")
def lib():
    out = os.path.join(ROOT, "build", "host_selftest_wiring.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    L = ctypes.CDLL(out)
    L.hs_permutation.restype = ctypes.c_int64
    L.hs_permutation.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return L


def host_permutation(lib, wL, wR, wO, n, m):
    """S1, S2, S3 (lists of ints) from the label body; the ids laid out as pb200_permutation takes them"""
    ids = np.full((n, 3), -1, dtype=np.int64)
    ids[:m, 0], ids[:m, 1], ids[:m, 2] = wL[:m], wR[:m], wO[:m]
    omega = np.frombuffer(pow(5, (R - 1) // n, R).to_bytes(32, "little"), dtype=np.uint32).copy()
    out = np.zeros(3 * n * 8, dtype=np.uint32)
    rc = lib.hs_permutation(ids.ctypes.data, n.bit_length() - 1, omega.ctypes.data, out.ctypes.data)
    assert rc == -1, rc
    raw = out.tobytes()
    vals = [int.from_bytes(raw[32 * k:32 * k + 32], "little") for k in range(3 * n)]
    return vals[:n], vals[n:2 * n], vals[2 * n:]


def check(lib, wL, wR, wO, n, m):
    got = host_permutation(lib, wL, wR, wO, n, m)
    want = syn.permutation_polys(wL, wR, wO, n, m)
    for k in range(3):
        assert list(got[k]) == list(want[k]), ("S%d" % (k + 1), n, m)
    return got


def test_reference_compiler_wirings(lib):
    """the wirings of the compiler entries of reference_vectors.json, rebuilt as test_synthetic_vs_reference does:
    equal to permutation_polys and to the reference compiler's digests"""
    for ref in load_json("reference_vectors.json")["compiler"]:
        log_n = ref["log_n"]
        c = syn.build_circuit(log_n, seed=log_n, n_public=2, fill=ref["fill"], with_text=True)
        S = check(lib, c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
        for k in range(3):
            assert digest(S[k]) == ref["polys"]["S%d" % (k + 1)], (log_n, k)


def random_wiring(rng, n, m, n_vars):
    w = [np.array([rng.randrange(-1, n_vars) for _ in range(n)], dtype=np.int64) for _ in range(3)]
    return w[0], w[1], w[2], n, m


@pytest.mark.parametrize("log_n", range(2, 13))
def test_random_wirings(lib, log_n):
    rng = random.Random(log_n)
    n = 1 << log_n
    for n_vars, m in ((2, n), (n, rng.randrange(1, n + 1)), (3 * n, n), (max(1, n // 4), rng.randrange(1, n + 1))):
        check(lib, *random_wiring(rng, n, m, n_vars))


def edge_cases(n):
    rng = random.Random(n)
    full = lambda v: np.full(n, v, dtype=np.int64)  # noqa: E731
    distinct = np.arange(3 * n, dtype=np.int64).reshape(n, 3)
    big = np.array([MAX_ID - rng.randrange(4) for _ in range(3 * n)], dtype=np.int64).reshape(n, 3)
    big[::5, 1] = -1
    return {
        "one variable": (full(7), full(7), full(7), n, n),
        "all distinct": (distinct[:, 0], distinct[:, 1], distinct[:, 2], n, n),
        "all unused": (full(-1), full(-1), full(-1), n, n),
        "one constraint": (full(3), full(4), full(3), n, 1),
        "ids up to 2^32 - 2": (big[:, 0], big[:, 1], big[:, 2], n, n),
        "ids 0 and 2^32 - 2": (full(0), full(MAX_ID), full(0), n, n // 2),
    }


@pytest.mark.parametrize("n", [2, 4, 64, 1024])
def test_edge_cases(lib, n):
    for name, case in edge_cases(n).items():
        check(lib, *case)


def test_host_check_names_the_first_bad_id(lib):
    n = 8
    for bad, cell in ((-2, 5), (MAX_ID + 1, 0), (1 << 40, 23)):
        ids = np.zeros(3 * n, dtype=np.int64)
        ids[cell] = bad
        ids[cell + 1:] = -7
        out = np.zeros(3 * n * 8, dtype=np.uint32)
        assert lib.hs_permutation(ids.ctypes.data, 3, None, out.ctypes.data) == cell


# ---- wiring.permutation_arrays refuses bad input before it touches the library -------------------------------------
@pytest.fixture
def no_library(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("the library was called")
    monkeypatch.setattr(wiring, "lib", refuse)
    monkeypatch.setattr(wiring, "default_context", refuse)


def wires(n, dtype=np.int64):
    return [np.arange(n, dtype=dtype) for _ in range(3)]


def test_refuses_id_below_minus_one(no_library):
    L, R_, O = wires(8)
    R_[3] = -2
    with pytest.raises(ValueError, match=r"wire_R\[3\] = -2"):
        wiring.permutation_arrays(L, R_, O, 8)


@pytest.mark.parametrize("bad", [MAX_ID + 1, 1 << 40])
def test_refuses_id_above_max(no_library, bad):
    L, R_, O = wires(8)
    O[6] = bad
    with pytest.raises(ValueError, match=r"wire_O\[6\] = %d" % bad):
        wiring.permutation_arrays(L, R_, O, 8)
    L, R_, O = wires(8, np.uint64)
    L[2] = np.uint64((1 << 64) - 1)
    with pytest.raises(ValueError, match=r"wire_L\[2\]"):
        wiring.permutation_arrays(L, R_, O, 8)


def test_refuses_wrong_length(no_library):
    L, R_, O = wires(8)
    with pytest.raises(ValueError, match="wire_L must be a 1-D array"):
        wiring.permutation_arrays(L[:7], R_, O, 8)
    with pytest.raises(ValueError, match="wire_O must be a 1-D array"):
        wiring.permutation_arrays(L[:5], R_[:5], O[:4], 8, n_constraints=5)
    with pytest.raises(ValueError, match="wire_R must be a 1-D array"):
        wiring.permutation_arrays(L, R_.reshape(2, 4), O, 8)


@pytest.mark.parametrize("dtype", [np.float64, np.bool_, object, np.str_])
def test_refuses_non_integer_dtype(no_library, dtype):
    L, R_, O = wires(8)
    with pytest.raises(ValueError, match="wire_L must hold integer variable ids"):
        wiring.permutation_arrays(L.astype(dtype), R_, O, 8)


@pytest.mark.parametrize("n", [0, 1, 3, 12, 1 << 27, 8.0, True])
def test_refuses_group_order_not_a_power_of_two(no_library, n):
    with pytest.raises(ValueError, match="group_order must be a power of two"):
        wiring.permutation_arrays(*wires(8), n)


@pytest.mark.parametrize("m", [-1, 9, 2.0])
def test_refuses_bad_n_constraints(no_library, m):
    with pytest.raises(ValueError, match="n_constraints must be an integer"):
        wiring.permutation_arrays(*wires(8), 8, n_constraints=m)


def test_accepts_valid_input_then_calls_the_library(no_library):
    """a valid wiring of any integer dtype, of length n_constraints or n, gets past the checks to the library"""
    for dtype in (np.int8, np.int32, np.int64, np.uint32, np.uint64):
        for length in (5, 8):
            w = np.arange(length, dtype=dtype)
            with pytest.raises(AssertionError, match="the library was called"):
                wiring.permutation_arrays(w, w, w, 8, n_constraints=5)
    # rows from n_constraints on are unused: whatever they hold is not checked
    w = np.full(8, -9, dtype=np.int64)
    w[:5] = 1
    with pytest.raises(AssertionError, match="the library was called"):
        wiring.permutation_arrays(w, w, w, 8, n_constraints=5)
