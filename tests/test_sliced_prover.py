"""Sliced round 3: a one-GPU prover whose cache on the 4n coset does not fit the device evaluates the quotient one
n-point slice of the coset at a time (csrc/memory_plan.cuh, "sliced round 3" in csrc/prover.cu).

CPU: the memory planner's choices and its count against DESIGN.md section 2.  GPU (PB200_SLICED=1 forces the sliced
path): the same bytes as the full path on both public-input paths, with and without custom terms; the golden proofs
reproduced; the features a sliced prover refuses are refused and leave it usable.  Opt-in (PB200_TEST_2P24=1): a
2^24-gate proof on one H100, which only fits sliced."""
import ctypes
import hashlib
import json
import os
import subprocess

import numpy as np
import pytest

from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from tests.golden_io import GOLDEN, PTAU_HEAD, ints, load_circuit

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
R = O.R_MOD
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
PK = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")
ALL_TERMS = [(2, 0, 0), (0, 0, 3), (2, 1, 0), (1, 1, 1)]
GB = 10 ** 9


# ---- CPU: the planner ----------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def hs():
    out = os.path.join(ROOT, "build", "host_selftest_plan.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    deps = [src] + [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith(".cuh")]
    if not os.path.exists(out) or any(os.path.getmtime(d) > os.path.getmtime(out) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    L = ctypes.CDLL(out)
    L.hs_prover_memory.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint64,
                                   ctypes.c_uint64, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]
    return L


def plan(hs, log_n, free, n_custom=0, force=False, msm_now=0):
    """(choice, full counts, sliced counts) for the fixed-base MSM the SRS of 2^log_n powers has (c = log_n, at most
    21 bits; three commitments per call)"""
    out = (ctypes.c_uint64 * 8)()
    choice = hs.hs_prover_memory(log_n, n_custom, min(max(log_n, 4), 21), 3, msm_now, int(free), int(force), out)
    return choice, list(out[:4]), list(out[4:])


@pytest.mark.parametrize("log_n", [20, 22])
def test_planner_keeps_the_full_path_when_it_fits(hs, log_n):
    choice, full, sliced = plan(hs, log_n, 80 * GB)
    assert choice == 0
    assert sum(sliced) < sum(full)
    assert plan(hs, log_n, 80 * GB, force=True)[0] == 1  # the knob forces slicing ...


def test_planner_slices_at_2p24(hs):
    choice, full, sliced = plan(hs, 24, 80 * GB)
    assert choice == 1
    assert sum(full) > 80 * GB - 4 * 2 ** 30 >= sum(sliced)


def test_planner_refuses_at_2p26(hs):
    choice, full, sliced = plan(hs, 26, 80 * GB)
    assert choice == -1
    assert plan(hs, 26, 80 * GB, force=True)[0] == -1  # ... and cannot make room


def test_planner_full_count_matches_design(hs):
    """DESIGN.md section 2: a per-circuit cache of 62n elements and a per-proof working set of about 40n"""
    n = 1 << 20
    _, full, _ = plan(hs, 20, 80 * GB)
    assert full[0] == 62 * n * 32
    assert abs(full[1] / (n * 32) - 40) <= 4
    # each custom term adds its selector three ways (6n) to the full cache and two ways plus one slice (3n) sliced
    _, full4, sliced4 = plan(hs, 20, 80 * GB, n_custom=4)
    _, _, sliced = plan(hs, 20, 80 * GB)
    assert full4[0] - full[0] == 4 * 6 * n * 32 and sliced4[0] - sliced[0] == 4 * 3 * n * 32


def test_planner_counts_only_msm_scratch_growth(hs):
    _, full, _ = plan(hs, 20, 80 * GB)
    _, grown, _ = plan(hs, 20, 80 * GB, msm_now=full[3])
    assert full[3] > 0 and grown[3] == 0 and grown[:3] == full[:3]


# ---- GPU -----------------------------------------------------------------------------------------------------------
@pytest.fixture
def sliced_env(monkeypatch):
    monkeypatch.setenv("PB200_SLICED", "1")
    return monkeypatch


def _circuit(log_n, n_public, terms, seed):
    """the synthetic circuit of the first seed from ``seed`` on whose rows use every term (small circuits may miss one)"""
    while True:
        c = syn.build_circuit(log_n, seed=seed, n_public=n_public, custom=terms)
        if all(any(col) for _, col in c.custom):
            return c
        seed += 1000


def _prover(pb, setup, n, pk, custom, sliced, monkeypatch):
    if sliced:
        monkeypatch.setenv("PB200_SLICED", "1")
    else:
        monkeypatch.delenv("PB200_SLICED", raising=False)
    prover = pb.Prover.from_arrays(setup, n, pk, custom=custom)
    assert prover.sliced == sliced
    return prover


@pytest.mark.gpu
@pytest.mark.parametrize("terms", [[], ALL_TERMS], ids=["plain", "all4"])
@pytest.mark.parametrize("log_n,n_public", [(4, 2), (8, 2), (12, 2), (4, 9), (8, 11), (12, 9)])
def test_sliced_equals_full(monkeypatch, terms, log_n, n_public):
    """<= 8 public inputs: PI from the closed-form basis on each slice; > 8: PI extended like A, B, C"""
    import plonkathon_b200 as pb
    c = _circuit(log_n, n_public, terms, 300 + log_n + n_public)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    custom = syn.custom_arrays(c)
    full = _prover(pb, setup, n, pk, custom, False, monkeypatch).prove_arrays(A, B, C, public)
    sliced = _prover(pb, setup, n, pk, custom, True, monkeypatch)
    assert sliced.prove_arrays(A, B, C, public) == full
    assert sliced.prove_arrays(A, B, C, public) == full  # state reuse


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["prover_test", "factorization", "poseidon"])
def test_sliced_golden_circuits(sliced_env, name):
    """prover_test is the reference's test/proof.pickle"""
    import plonkathon_b200 as pb
    entry, arr = load_circuit(name)
    setup = pb.Setup.from_file(PTAU_HEAD)
    prover = pb.Prover.from_arrays(setup, entry["n"], {k: arr[k] for k in PK})
    assert prover.sliced
    raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"]


@pytest.mark.gpu
def test_sliced_golden_custom_proof_2p16(sliced_env):
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_custom_2p16.json")))
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"],
                          custom=[tuple(e) for e in rec["terms"]])
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    prover = pb.Prover.from_arrays(pb.Setup.generate(TAU, n), n, pk, custom=syn.custom_arrays(c))
    assert prover.sliced
    assert prover.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]


@pytest.mark.gpu
def test_sliced_golden_2p20_and_full_by_default(monkeypatch):
    import plonkathon_b200 as pb
    log_n = 20
    n = 1 << log_n
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    c = syn.build_circuit(log_n, seed=rec["seed"], n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n)
    monkeypatch.delenv("PB200_SLICED", raising=False)
    assert not pb.Prover.from_arrays(setup, n, pk).sliced  # the full path fits an H100 at 2^20
    prover = _prover(pb, setup, n, pk, (), True, monkeypatch)
    raw = prover.prove_arrays(A, B, C, public)
    assert raw.hex() == rec["proof_hex"], "sliced proof differs from the oracle's golden proof at 2^20 gates"


@pytest.mark.gpu
def test_sliced_prover_refuses_whole_coset_features(sliced_env):
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    entry, arr = load_circuit("factorization")
    n = entry["n"]
    setup = pb.Setup.from_file(PTAU_HEAD)
    prover = pb.Prover.from_arrays(setup, n, {k: arr[k] for k in PK})
    assert prover.sliced
    L = _lib.lib()
    col = np.zeros((n, 32), np.uint8)
    p = col.ctypes.data_as(ctypes.c_void_p)
    calls = {
        "set_zk": lambda: L.pb200_prover_set_zk(prover._h, 1, None),
        "set_zk_lookup": lambda: L.pb200_prover_set_zk_lookup(prover._h, 1, None),
        "set_zk_shuffle": lambda: L.pb200_prover_set_zk_shuffle(prover._h, 1, None),
        "set_lookup": lambda: L.pb200_prover_set_lookup(prover._h, p, p, p, p, 1),
        "set_lookup_tagged": lambda: L.pb200_prover_set_lookup_tagged(prover._h, p, p, p, p, p, p, 1),
        "set_shuffle": lambda: L.pb200_prover_set_shuffle(prover._h, p, p),
    }
    for what, call in calls.items():
        assert call() != 0, what
        assert "sliced prover" in L.pb200_last_error().decode(), what
        raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
        assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"], what
    assert L.pb200_prover_set_zk(prover._h, 0, None) == 0  # switching it off is not an error
    with pytest.raises(_lib.PlonkB200Error, match="sliced prover.*next-row"):
        pb.Prover.from_arrays(setup, n, {k: arr[k] for k in PK}, custom=[((1, 0, 0, 0, 1, 0), arr["QL"])])


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("PB200_TEST_2P24") != "1",
                    reason="opt-in (PB200_TEST_2P24=1): a 2^24-gate proof on one H100, minutes of host work")
def test_prove_2p24_gates_sliced(monkeypatch):
    """2^24 gates: the full path does not fit 80 GB, so the prover slices without the knob.  No golden: the oracle
    would take hours; the proof is checked by both verifier routines and by the trapdoor verifier instead."""
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    monkeypatch.delenv("PB200_SLICED", raising=False)
    log_n = 24
    n = 1 << log_n
    c = syn.build_circuit(log_n, seed=7, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    del c
    setup = pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk)
    assert prover.sliced
    raw = prover.prove_arrays(A, B, C, public)
    assert prover.prove_arrays(A, B, C, public) == raw
    pub_ints = [int(x) for x in public]
    del prover
    pvk = setup.verification_key_arrays(n, pk)
    assert pvk.verify_proof(n, pb.Proof.from_bytes(raw), pub_ints)
    assert pvk.verify_proof_unoptimized(n, pb.Proof.from_bytes(raw), pub_ints)

    def commit(col):
        out = ctypes.create_string_buffer(64)
        ident = ctypes.c_int()
        _lib.check(_lib.lib().pb200_srs_commit_lagrange_host(
            setup.ctx.handle, setup._srs, pk[col].ctypes.data_as(ctypes.c_void_p), log_n, out, ctypes.byref(ident)))
        return None if ident.value else (int.from_bytes(out.raw[:32], "little"), int.from_bytes(out.raw[32:], "little"))

    vk = {k: commit(col) for k, col in (("Qm", "QM"), ("Ql", "QL"), ("Qr", "QR"), ("Qo", "QO"), ("Qc", "QC"),
                                        ("S1", "S1"), ("S2", "S2"), ("S3", "S3"))}
    proof = O.proof_from_bytes(raw)
    assert O.verify_proof_trapdoor(n, vk, proof, public, TAU)
    bad = dict(proof)
    bad["z_shifted_eval"] = (bad["z_shifted_eval"] + 1) % R
    assert not O.verify_proof_trapdoor(n, vk, bad, public, TAU)
    k = 32 * 19  # z_shifted_eval in the 768 bytes
    raw_bad = raw[:k] + ((int.from_bytes(raw[k:k + 32], "big") + 1) % R).to_bytes(32, "big") + raw[k + 32:]
    assert not pvk.verify_proof(n, pb.Proof.from_bytes(raw_bad), pub_ints)
    assert not pvk.verify_proof_unoptimized(n, pb.Proof.from_bytes(raw_bad), pub_ints)
