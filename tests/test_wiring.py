"""GPU: wiring.permutation_arrays (csrc/permutation.cu) against synthetic.permutation_polys, the CPU restatement of the
reference compiler's permutation, byte for byte: the reference compiler's wirings (and its digests), random wirings,
the edge cases, and bench-family circuits with custom, lookup and shuffle rows.  A proving key built on the GPU's
S1..S3 reproduces the golden 2^20-gate proof, and a refused call leaves the context usable."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest

from plonkathon_b200 import synthetic as syn
from tests.golden_io import GOLDEN, PTAU_HEAD, digest, ints, load_circuit, load_json
from tests.test_wiring_host import edge_cases, random_wiring

pytestmark = pytest.mark.gpu

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
R = syn.R
PK = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")


def le(vals):
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in vals), dtype=np.uint8).reshape(-1, 32)


def gpu(wL, wR, wO, n, m):
    from plonkathon_b200 import permutation_arrays
    S = permutation_arrays(wL, wR, wO, n, n_constraints=m)
    assert all(S[k].shape == (n, 32) and S[k].dtype == np.uint8 for k in ("S1", "S2", "S3"))
    return S


def check(wL, wR, wO, n, m):
    S = gpu(wL, wR, wO, n, m)
    want = syn.permutation_polys(wL, wR, wO, n, m)
    for k in range(3):
        assert np.array_equal(S["S%d" % (k + 1)], le(want[k])), ("S%d" % (k + 1), n, m)
    return S


def test_reference_compiler_wirings():
    for ref in load_json("reference_vectors.json")["compiler"]:
        log_n = ref["log_n"]
        c = syn.build_circuit(log_n, seed=log_n, n_public=2, fill=ref["fill"], with_text=True)
        S = check(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
        for k in range(3):
            assert hashlib.sha256(S["S%d" % (k + 1)].tobytes()).hexdigest() == ref["polys"]["S%d" % (k + 1)]


@pytest.mark.parametrize("log_n", range(2, 13))
def test_random_wirings(log_n):
    rng = random.Random(log_n)
    n = 1 << log_n
    for n_vars, m in ((2, n), (n, rng.randrange(1, n + 1)), (3 * n, n), (max(1, n // 4), rng.randrange(1, n + 1))):
        check(*random_wiring(rng, n, m, n_vars))


@pytest.mark.parametrize("n", [2, 4, 64, 1024])
def test_edge_cases(n):
    for name, case in edge_cases(n).items():
        check(*case)


def test_two_calls_give_the_same_bytes():
    c = syn.build_circuit(14, seed=5, n_public=2, shuffle=True)
    a = gpu(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
    b = gpu(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)
    assert all(np.array_equal(a[k], b[k]) for k in a)


def range_table(n):
    k = max(2, n // 2)
    return [list(range(k)), [0] * k, [0] * k]


CIRCUITS = {
    "plain": {},
    "custom": {"custom": [(2, 1, 0), (0, 1, 2), (1, 1, 1)]},
    "next-row custom, shuffle": {"custom": [(0, 0, 0, 1, 0, 0), (0, 1, 1, 0, 0, 1)], "shuffle": True},
    "lookup": {"lookup": None},
    "lookups": {"lookups": None},
    "shuffle": {"shuffle": True},
}


@pytest.mark.parametrize("log_n,kind", [(16, k) for k in CIRCUITS] + [(20, k) for k in ("plain", "lookup", "shuffle")])
def test_bench_family_circuits(log_n, kind):
    kw = dict(CIRCUITS[kind])
    if "lookup" in kw:
        kw["lookup"] = range_table(1 << 10)
    if "lookups" in kw:
        kw["lookups"] = [range_table(1 << 8), [[1, 2, 3], [4, 5, 6], [7, 8, 9]]]
    c = syn.build_circuit(log_n, seed=7, n_public=2, **kw)
    check(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)


def test_golden_2p20_proof_from_gpu_permutation():
    """S1..S3 from the GPU in the pk arrays of the 2^20 circuit of proof_2p20.json: the golden proof byte for byte, and
    the key from the same arrays verifies it with both routines"""
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    log_n = rec["log_n"]
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=rec["seed"], n_public=rec["n_public"])
    sel = {k: le(getattr(c, k)) for k in PK[:5]}
    A, B, C = (le(w) for w in c.wires_values())
    public = c.public_values()
    pk = dict(sel, **pb.permutation_arrays(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints))
    setup = pb.Setup.generate(TAU, n)
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(A, B, C, public)
    assert raw.hex() == rec["proof_hex"]
    vk = setup.verification_key_arrays(n, pk)
    assert (vk.S1[0].n, vk.S1[1].n) == tuple(int(x) for x in rec["vk"]["S1"])
    assert (vk.S3[0].n, vk.S3[1].n) == tuple(int(x) for x in rec["vk"]["S3"])
    pub = [int(x) for x in public]
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), pub)
    assert vk.verify_proof_unoptimized(n, pb.Proof.from_bytes(raw), pub)


def test_refused_calls_leave_the_context_usable():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    L = _lib.lib()
    ctx = pb.default_context()
    n = 16
    out = np.zeros(3 * n * 32, np.uint8)
    ids = np.zeros(3 * n, np.int64)
    for bad, cell, text in ((-2, 7, "cell 7 (row 2, wire R)"), ((1 << 32) - 1, 47, "cell 47 (row 15, wire O)")):
        ids[:] = 0
        ids[cell] = bad
        assert L.pb200_permutation(ctx.handle, ids.ctypes.data_as(ctypes.c_void_p), 4,
                                   out.ctypes.data_as(ctypes.c_void_p)) != 0
        assert text in L.pb200_last_error().decode()
    ids[:] = 0
    for log_n in (0, 27, -1):
        assert L.pb200_permutation(ctx.handle, ids.ctypes.data_as(ctypes.c_void_p), log_n,
                                   out.ctypes.data_as(ctypes.c_void_p)) != 0
        assert "1 <= k <= 26" in L.pb200_last_error().decode()
    assert not out.any()  # nothing written by a refused call
    # a proof right after, and the permutation itself
    entry, arr = load_circuit("factorization")
    setup = pb.Setup.from_file(PTAU_HEAD)
    raw = pb.Prover.from_arrays(setup, entry["n"], {k: arr[k] for k in PK}).prove_arrays(
        arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"]
    c = syn.build_circuit(10, seed=3, n_public=2)
    check(c.wire_L, c.wire_R, c.wire_O, c.group_order, c.n_constraints)


@pytest.mark.skipif(os.environ.get("PB200_TEST_2P24") != "1",
                    reason="opt-in (PB200_TEST_2P24=1): a 2^24-gate circuit, minutes of host work")
def test_2p24_gpu_permutation_proves():
    """2^24 gates: the GPU's S1..S3 equal the CPU reference, and a proof on them verifies"""
    import plonkathon_b200 as pb
    log_n = 24
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=7, n_public=2)
    S = gpu(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    want = syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)
    for k in range(3):
        assert hashlib.sha256(S["S%d" % (k + 1)].tobytes()).hexdigest() == digest(want[k]), k
    del want
    pk = dict({k: le(getattr(c, k)) for k in PK[:5]}, **S)
    A, B, C = (le(w) for w in c.wires_values())
    public = [int(x) for x in c.public_values()]
    del c
    setup = pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk)
    raw = prover.prove_arrays(A, B, C, public)
    del prover
    vk = setup.verification_key_arrays(n, pk)
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), public)
    assert vk.verify_proof_unoptimized(n, pb.Proof.from_bytes(raw), public)
    bad = raw[:32 * 19] + ((int.from_bytes(raw[32 * 19:32 * 20], "big") + 1) % R).to_bytes(32, "big") + raw[32 * 20:]
    assert not vk.verify_proof(n, pb.Proof.from_bytes(bad), public)
