"""GPU: the witness check (``Prover.check_arrays``, csrc/check.cu) against the independent CPU checker
(tests/witness_check.py) and against proving.

Valid witnesses give empty reports: the three golden circuits, the eight 2^16 golden feature circuits, the 2^20 golden
circuit and the sliced prover.  Planted faults give the CPU checker's counts and lists on every proof kind at 2^4, 2^8
and 2^12 on both public-input paths, and ``prove_arrays`` raises AssertionError on each; at 2^20 a thousand mixed faults
give exact counts and the lowest 16 of each.  A check leaves the round state and every later proof unchanged, the device
entry point equals the host one, and refused calls leave the prover proving.  Opt-in (PB200_TEST_2P24=1): a 2^24 sliced
prover."""
import ctypes
import hashlib
import json
import os
import random

import numpy as np
import pytest

from plonkathon_b200 import synthetic as syn
from tests import witness_check as WC
from tests.golden_io import GOLDEN, ints, load_circuit
from tests.test_check_host import KINDS, kind_circuit

R = WC.R
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
PK = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")
PTAU_HEAD = os.path.join(GOLDEN, "powersOfTau28_hez_final_11.head.ptau")
NAMES = ("gate", "copy", "key", "lookup", "shuffle")

pytestmark = pytest.mark.gpu


def _le(ints_):
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in ints_), np.uint8).reshape(-1, 32).copy()


def _prover(pb, c, setup=None, S=None, extra=0):
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    if S is not None:
        pk.update(S1=_le(S[0]), S2=_le(S[1]), S3=_le(S[2]))
    kw = {}
    if c.custom:
        kw["custom"] = syn.custom_arrays(c)
    if c.shuffle:
        kw["shuffle"] = syn.shuffle_arrays(c)
    if c.lookup:
        kw["lookup"] = syn.lookup_arrays(c)
    if c.lookups:
        kw["lookups"] = syn.lookups_arrays(c)
    setup = setup or pb.Setup.generate(TAU, n + extra)
    return setup, pb.Prover.from_arrays(setup, n, pk, **kw), pk


def _as_cpu(rep):
    return {"counts": [getattr(rep, k) for k in NAMES], "gate": rep.gate_rows, "copy": rep.copy_pairs,
            "key": rep.key_cells, "lookup": rep.lookup_rows, "shuffle": rep.shuffle_rows}


# ---- valid witnesses -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["prover_test", "factorization", "poseidon"])
def test_golden_circuits_are_clean(name):
    import plonkathon_b200 as pb
    entry, arr = load_circuit(name)
    prover = pb.Prover.from_arrays(pb.Setup.from_file(PTAU_HEAD), entry["n"], {k: arr[k] for k in PK})
    rep = prover.check_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    assert rep.ok, str(rep)
    raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
    assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"]


FEATURES = ["custom", "zk", "next_row", "shuffle", "zk_shuffle", "lookup", "tagged_lookup", "zk_lookup"]


@pytest.mark.parametrize("kind", FEATURES)
def test_feature_goldens_2p16_are_clean_and_prove_unchanged(kind):
    """zero-knowledge kinds with the record's fixed blinders: the proof after the check is the golden"""
    import plonkathon_b200 as pb
    from tests.golden import make_feature_proofs_2p16 as G
    make, _, extra, _ = G.KINDS[kind]
    rec = json.load(open(os.path.join(GOLDEN, "proof_%s_2p16.json" % kind)))
    c = make()
    _, prover, _ = _prover(pb, c, extra=extra)
    if kind.startswith("zk"):
        {"zk": prover.set_zk, "zk_shuffle": prover.set_zk_shuffle, "zk_lookup": prover.set_zk_lookup}[kind](
            True, [int(b) for b in rec["blinders"]])
    A, B, C = (_le(x) for x in c.wires_values())
    public = c.public_values()
    rep = prover.check_arrays(A, B, C, public)
    assert rep.ok, str(rep)
    assert prover.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]


def test_golden_2p20_is_clean_and_a_check_over_its_memory_cap_is_refused(monkeypatch):
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    c = syn.build_circuit(20, seed=rec["seed"], n_public=2)
    setup, prover, pk = _prover(pb, c)
    A, B, C = (_le(x) for x in c.wires_values())
    public = c.public_values()
    # a cap below what the first check needs (sigma's build, 56 bytes a cell): refused before any device work, naming
    # the bytes; without the cap the same call succeeds
    monkeypatch.setenv("PB200_CHECK_MAX_BYTES", str(100 << 20))
    with pytest.raises(_lib.PlonkB200Error, match=r"witness check of 2\^20 rows needs \d+ bytes of device memory, "
                                                   r"104857600 are free"):
        prover.check_arrays(A, B, C, public)
    monkeypatch.delenv("PB200_CHECK_MAX_BYTES")
    rep = prover.check_arrays(A, B, C, public)
    assert rep.ok, str(rep)
    assert prover.prove_arrays(A, B, C, public).hex() == rec["proof_hex"]


def test_device_wires_written_on_a_torch_stream_are_read_after_the_writes():
    """the wires reach their tensors on a side stream behind a long queue of work; check_arrays must see them"""
    import torch
    import plonkathon_b200 as pb
    c = kind_circuit("plain", 16)
    _, prover, _ = _prover(pb, c)
    host = [torch.from_numpy(_le(x)).pin_memory() for x in c.wires_values()]
    public = c.public_values()
    dev = [torch.zeros_like(h, device="cuda") for h in host]  # zero wires fail the constant gates
    assert not prover.check_arrays(*dev, public).ok
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        x = torch.randn(4096, 4096, device="cuda")
        for _ in range(20):  # keep the side stream busy well past the call below
            x = x @ x / 64
        for d, h in zip(dev, host):
            d.copy_(h, non_blocking=True)
        rep = prover.check_arrays(*dev, public)
    assert rep.ok, str(rep)


def test_sliced_prover(monkeypatch):
    import plonkathon_b200 as pb
    monkeypatch.setenv("PB200_SLICED", "1")
    c = kind_circuit("custom", 12, n_public=9)
    _, prover, _ = _prover(pb, c)
    assert prover.sliced
    A, B, C = c.wires_values()
    public = c.public_values()
    assert prover.check_arrays(A, B, C, public).ok
    bad = list(C)
    for r in (100, 2000, 4000):
        bad[r] = (bad[r] + 1) % R
    assert _as_cpu(prover.check_arrays(A, B, bad, public)) == WC.check_circuit(c, A, B, bad, public)
    with pytest.raises(AssertionError):
        prover.prove_arrays(A, B, bad, public)


# ---- planted faults --------------------------------------------------------------------------------------------------
def _planted(c, rng):
    """(name, A, B, C, public) faulted witnesses of c, and a key fault as (name, S) pairs"""
    from tests.test_check_host import faults
    n = c.group_order
    out = faults(c, rng)[1:]
    A, B, C = (list(x) for x in c.wires_values())
    public = c.public_values()
    if c.lookups:  # a tagged row set to a row of another table only
        tables = [list(zip(*t)) for _, t in c.lookups]
        for i in range(n):
            own = [k for k, (q, _) in enumerate(c.lookups) if q[i]]
            if own:
                other = [row for k, t in enumerate(tables) if k != own[0] for row in t if row not in tables[own[0]]]
                if other:
                    a, b, cc = other[0]
                    out.append(("tagged", A[:i] + [a] + A[i + 1:], B[:i] + [b] + B[i + 1:], C[:i] + [cc] + C[i + 1:],
                                public))
                    break
    if n >= 256:  # more faults than the limit
        bad = list(C)
        for r in rng.sample(range(c.n_public, n), 40):
            bad[r] = (bad[r] + 1) % R
        out.append(("many", A, B, bad, public))
    S = [list(s) for s in syn.permutation_polys(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints)]
    dup, non = [s[:] for s in S], [s[:] for s in S]
    dup[1][3] = S[1][1]
    non[1][3] = 12345
    return out, [("duplicate label", dup), ("non-label", non)]


@pytest.mark.parametrize("log_n,n_public", [(4, 2), (8, 2), (12, 2), (8, 11), (12, 9)])
@pytest.mark.parametrize("kind", KINDS)
def test_planted_faults_equal_the_cpu_checker(kind, log_n, n_public):
    """<= 8 public inputs and > 8: the prover's two public-input paths"""
    import plonkathon_b200 as pb
    c = kind_circuit(kind, log_n, n_public=n_public)
    setup, prover, _ = _prover(pb, c)
    rng = random.Random(log_n * 100 + n_public + KINDS.index(kind))
    witnesses, keys = _planted(c, rng)
    A, B, C = c.wires_values()
    public = c.public_values()
    assert prover.check_arrays(A, B, C, public).ok
    for name, fa, fb, fc, fp in witnesses:
        rep = prover.check_arrays(fa, fb, fc, fp)
        assert not rep.ok, name
        assert _as_cpu(rep) == WC.check_circuit(c, fa, fb, fc, fp), name
        with pytest.raises(AssertionError):
            prover.prove_arrays(fa, fb, fc, fp)
    good = prover.prove_arrays(A, B, C, public)  # every failed proof left the prover proving
    assert prover.check_arrays(A, B, C, public).ok
    for name, S in keys:
        _, kp, _ = _prover(pb, c, setup, S=S)
        rep = kp.check_arrays(A, B, C, public)
        want = WC.check_circuit(c, A, B, C, public, S=S)
        assert _as_cpu(rep) == want and rep.key >= 1, name
        with pytest.raises(AssertionError):
            kp.prove_arrays(A, B, C, public)
    assert prover.prove_arrays(A, B, C, public) == good


def test_a_thousand_mixed_faults_at_2p20():
    import plonkathon_b200 as pb
    c = syn.build_circuit(20, seed=7, n_public=2, shuffle=True)
    n = c.group_order
    _, prover, _ = _prover(pb, c)
    A, B, C = (list(x) for x in c.wires_values())
    public = c.public_values()
    rng = random.Random(1000)
    W = [A, B, C]
    for cell in rng.sample(range(3 * n), 1000):
        row, col = divmod(cell, 3)
        W[col][row] = (W[col][row] + rng.randrange(1, 1000)) % R
    rep = prover.check_arrays(A, B, C, public, limit=16)
    want = WC.check_circuit(c, A, B, C, public, limit=16)
    assert _as_cpu(rep) == want
    assert all(rep.counts()[k] >= 16 for k in ("gate", "copy", "shuffle")), rep.counts()


# ---- state -------------------------------------------------------------------------------------------------------------
def test_check_between_rounds_leaves_the_proof_unchanged():
    import plonkathon_b200 as pb
    from plonkathon_b200.transcript import Transcript
    c = kind_circuit("custom", 8)
    _, prover, _ = _prover(pb, c)
    A, B, C = (_le(x) for x in c.wires_values())
    public = c.public_values()
    whole = prover.prove_arrays(A, B, C, public)
    tr = Transcript(b"plonk")
    msg_1 = prover.round_1_arrays(A, B, C, public)
    bad = C.copy()
    bad[50, 0] ^= 1
    assert not prover.check_arrays(A, B, bad, public).ok  # a failing witness, between round 1 and round 2
    assert prover.check_arrays(A, B, C, public).ok
    prover.beta, prover.gamma = tr.round_1(msg_1, prover._kind.schedule)
    msg_2 = prover.round_2()
    prover.alpha, prover.fft_cofactor = tr.round_2(msg_2)
    msg_3 = prover.round_3()
    prover.zeta = tr.round_3(msg_3)
    msg_4 = prover.round_4()
    prover.v = tr.round_4(msg_4)
    msg_5 = prover.round_5()
    assert pb.Proof(msg_1, msg_2, msg_3, msg_4, msg_5).to_bytes() == whole


@pytest.mark.parametrize("kind", ["plain", "next_row_shuffle", "tagged"])
def test_device_entry_point_equals_the_host_one(kind):
    import torch
    import plonkathon_b200 as pb
    c = kind_circuit(kind, 10)
    _, prover, _ = _prover(pb, c)
    A, B, C = (list(x) for x in c.wires_values())
    rng = random.Random(3)
    for cell in rng.sample(range(3 * c.group_order), 50):
        row, col = divmod(cell, 3)
        [A, B, C][col][row] = ([A, B, C][col][row] + 1) % R
    public = c.public_values()
    host = prover.check_arrays(A, B, C, public, limit=8)
    dev = prover.check_arrays(*[torch.from_numpy(_le(x)).cuda() for x in (A, B, C)], public, limit=8)
    assert _as_cpu(dev) == _as_cpu(host) and not host.ok
    assert str(dev) == str(host)


def test_refusals_leave_the_prover_proving():
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    c = kind_circuit("shuffle", 8)
    setup, prover, pk = _prover(pb, c)
    A, B, C = (_le(x) for x in c.wires_values())
    public = c.public_values()
    good = prover.prove_arrays(A, B, C, public)
    bad = A.copy()
    bad[7] = np.frombuffer(R.to_bytes(32, "little"), np.uint8)
    with pytest.raises(_lib.PlonkB200Error, match="wire value not reduced below the field modulus"):
        prover.check_arrays(bad, B, C, public)
    L = _lib.lib()
    counts, lists = (ctypes.c_uint64 * 5)(), (ctypes.c_uint32 * 6)()
    pub = np.frombuffer(R.to_bytes(32, "little"), np.uint8).reshape(1, 32).copy()
    ptr = lambda a: a.ctypes.data_as(ctypes.c_void_p)  # noqa: E731
    assert L.pb200_prover_check(prover._h, ptr(A), ptr(B), ptr(C), ptr(pub), 1, 1, counts, lists) != 0
    assert "public input not reduced below the field modulus" in L.pb200_last_error().decode()
    assert L.pb200_prover_check(prover._h, ptr(A), ptr(B), ptr(C), ptr(pub), 257, 1, counts, lists) != 0
    assert "more public inputs than rows" in L.pb200_last_error().decode()
    assert prover.prove_arrays(A, B, C, public) == good
    assert prover.check_arrays(A, B, C, public).ok
    # the sharded prover, on a communicator of one rank
    ctx = pb.Context(0)
    uid = ctypes.create_string_buffer(128)
    if L.pb200_comm_unique_id(uid) != 0 or L.pb200_comm_init(ctx.handle, uid, 0, 1) != 0:
        pytest.skip("no communicator here: %s" % L.pb200_last_error().decode())
    arr = (ctypes.c_char_p * 8)(*[pk[k].tobytes() for k in PK])
    h = ctypes.c_void_p()
    _lib.check(L.pb200_prover_create_sharded(ctx.handle, setup._srs, 8, ctypes.cast(arr, ctypes.c_void_p),
                                             ctypes.byref(h)))
    try:
        assert L.pb200_prover_check(h, ptr(A), ptr(B), ptr(C), None, 0, 1, counts, lists) != 0
        assert "not available on the sharded prover" in L.pb200_last_error().decode()
    finally:
        L.pb200_prover_destroy(h)
    assert prover.prove_arrays(A, B, C, public) == good


@pytest.mark.skipif(os.environ.get("PB200_TEST_2P24") != "1",
                    reason="opt-in (PB200_TEST_2P24=1): a 2^24-gate circuit on one H100, minutes of host work")
def test_check_2p24_sliced(monkeypatch):
    import plonkathon_b200 as pb
    monkeypatch.delenv("PB200_SLICED", raising=False)
    c = syn.build_circuit(24, seed=7, n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    prover = pb.Prover.from_arrays(pb.Setup.generate(TAU, n), n, pk)
    assert prover.sliced
    assert prover.check_arrays(A, B, C, public).ok
    rng = random.Random(24)
    rows = sorted(rng.sample(range(2, n), 300))
    changed = np.zeros(3 * n, dtype=bool)
    for r in rows:  # the output wire of 300 rows
        C[r, 0] ^= 1
        changed[3 * r + 2] = True
    gates = [r for r in rows if c.QO[r] % R]  # a changed output fails the rows whose gate reads it
    copies = WC.copy_failures(c.wire_L, c.wire_R, c.wire_O, n, c.n_constraints, changed)
    rep = prover.check_arrays(A, B, C, public)
    assert rep.counts() == {"gate": len(gates), "copy": len(copies), "key": 0, "lookup": 0, "shuffle": 0}
    assert rep.gate_rows == gates[:16] and rep.copy_pairs == [tuple(p) for p in copies[:16].tolist()]
