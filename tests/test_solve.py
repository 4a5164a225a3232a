"""Wire values from inputs (plonkathon_b200/solve.py, csrc/solve.cu): a Python restatement of the rule against the
reference compiler's ``fill_variable_assignments`` (tests/golden/solve_programs.json, make_solve_fixture.py), the shared
gate body run in row order on the CPU (csrc/host_selftest.cpp), the refusals, and on the GPU: the reference programs,
synthetic circuits of every proof kind, proofs from device-resident wires, the dependency paths and the errors."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pytest

from plonkathon_b200 import synthetic as syn
from plonkathon_b200.custom_gates import padded
from tests.golden_io import GOLDEN, load_circuit, load_json
from tests.test_check_host import KINDS, kind_circuit

R = syn.R
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "plonkathon_b200", "csrc")
SEL = ("QL", "QR", "QM", "QO", "QC")


def _le(ints_):
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in ints_), np.uint8).reshape(-1, 32).copy()


def _ints(arr):
    raw = np.ascontiguousarray(arr).tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


def _digest(ints_):
    return hashlib.sha256(b"".join(int(x).to_bytes(32, "little") for x in ints_)).hexdigest()


# ---- the restatement -------------------------------------------------------------------------------------------------
def _reads_c(e):
    e = padded(e)
    return e[2] > 0 or any(e[3:])


def defining_rows(ids, m, sel, custom, inputs):
    """{variable: its defining row} under the rule (solve.py's docstring); ids: (n, 3) int array"""
    out = {}
    for r in range(m):
        v = int(ids[r, 2])
        if v < 0 or sel["QO"][r] == 0 or v in inputs or v in out:
            continue
        if any(_reads_c(e) and col[r] for e, col in custom):
            continue
        out[v] = r
    return out


def restate(ids, n, m, sel, custom, inputs):
    """-> (A, B, C) as ints, or (unset cells, order (cell, row) pairs) when the rule leaves cells without a value"""
    ids = np.asarray(ids).reshape(n, 3)
    defs = defining_rows(ids, m, sel, custom, inputs)
    unset, order = [], []
    for c in range(3 * m):
        v = int(ids[c // 3, c % 3])
        if v >= 0 and v not in inputs and v not in defs:
            unset.append(c)
        r, col = divmod(c, 3)
        if col < 2 and defs.get(int(ids[r, 2])) == r and v in defs and defs[v] >= r:
            order.append((c, defs[v]))
    if unset or order:
        return None, unset, order
    val = {-1: 0}
    val.update(inputs)
    for r in range(m):
        v = int(ids[r, 2])
        if defs.get(v) != r:
            continue
        a, b = val[int(ids[r, 0])], val[int(ids[r, 1])]
        s = sel["QL"][r] * a + sel["QR"][r] * b + sel["QM"][r] * a * b + sel["QC"][r]
        for e, col in custom:
            e = padded(e)
            s += col[r] * pow(a, e[0], R) * pow(b, e[1], R) * (0 if any(e[2:]) else 1)
        val[v] = -s * pow(sel["QO"][r], R - 2, R) % R
    cols = [[val[int(ids[r, k])] if r < m else 0 for r in range(n)] for k in range(3)]
    return cols, [], []


def free_variables(c):
    """the inputs of a synthetic circuit: every variable in a cell that no row defines under the rule"""
    ids = np.stack([c.wire_L, c.wire_R, c.wire_O], axis=1)
    sel = {k: getattr(c, k) for k in SEL}
    defs = defining_rows(ids, c.n_constraints, sel, c.custom, {})
    used = {int(x) for x in ids[:c.n_constraints].reshape(-1) if x >= 0}
    return {v: c.values[v] for v in sorted(used - set(defs))}


def _program(name):
    e = load_json("solve_programs.json")[name]
    n, m = e["n"], e["n_constraints"]
    ids = np.full((n, 3), -1, np.int64)
    for k, w in enumerate(("wire_L", "wire_R", "wire_O")):
        ids[:m, k] = e[w]
    sel = {k: [int(x) % R for x in e["selectors"][k]] for k in SEL}
    inputs = {int(k): int(v) % R for k, v in e["inputs"].items()}
    return e, ids, n, m, sel, inputs


PROGRAMS = ["prover_test", "factorization", "poseidon"]


@pytest.mark.parametrize("name", PROGRAMS)
def test_restatement_reproduces_the_reference_fill(name):
    e, ids, n, m, sel, inputs = _program(name)
    cols, unset, order = restate(ids, n, m, sel, [], inputs)
    assert not unset and not order
    for k, col in zip("ABC", cols):
        assert _digest(col[:m]) == e["columns_sha256"][k], k


@pytest.mark.parametrize("kind", KINDS)
def test_restatement_reproduces_synthetic_wires(kind):
    c = kind_circuit(kind, 6)
    ids = np.stack([c.wire_L, c.wire_R, c.wire_O], axis=1)
    cols, unset, order = restate(ids, c.group_order, c.n_constraints, {k: getattr(c, k) for k in SEL}, c.custom,
                                 free_variables(c))
    assert (unset, order) == ([], [])
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())


@pytest.fixture(scope="module")
def hs():
    out = os.path.join(ROOT, "build", "host_selftest_solve.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    src = os.path.join(CSRC, "host_selftest.cpp")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", src, "-I", CSRC, "-o", out])
    return ctypes.CDLL(out)


def _hs_solve(hs, ids, n, m, sel, custom, inputs):
    vp = ctypes.c_void_p
    ids = np.ascontiguousarray(np.asarray(ids, np.int64).reshape(-1))
    s = np.concatenate([_le(sel[k]) for k in SEL])
    cust = np.concatenate([_le(col) for _, col in custom]) if custom else np.zeros((1, 32), np.uint8)
    exps = bytes(x for e, _ in custom for x in padded(e)) or b"\0"
    in_ids = np.array(list(inputs), np.int64)
    in_vals = _le(list(inputs.values())) if inputs else np.zeros((1, 32), np.uint8)
    out = np.zeros((3 * n, 32), np.uint8)
    rc = hs.hs_solve(ids.ctypes.data_as(vp), n.bit_length() - 1, ctypes.c_uint64(m), s.ctypes.data_as(vp), len(custom),
                     exps, cust.ctypes.data_as(vp), ctypes.c_uint64(len(in_ids)), in_ids.ctypes.data_as(vp),
                     in_vals.ctypes.data_as(vp), out.ctypes.data_as(vp))
    return rc, [_ints(out[k * n:(k + 1) * n]) for k in range(3)]


@pytest.mark.parametrize("name", PROGRAMS)
def test_shared_gate_body_reproduces_the_reference_fill(hs, name):
    e, ids, n, m, sel, inputs = _program(name)
    rc, cols = _hs_solve(hs, ids, n, m, sel, [], inputs)
    assert rc == 0
    for k, col in zip("ABC", cols):
        assert _digest(col[:m]) == e["columns_sha256"][k], k


@pytest.mark.parametrize("kind", ["custom", "next_row"])
def test_shared_gate_body_reproduces_synthetic_wires(hs, kind):
    c = kind_circuit(kind, 6)
    ids = np.stack([c.wire_L, c.wire_R, c.wire_O], axis=1)
    rc, cols = _hs_solve(hs, ids, c.group_order, c.n_constraints, {k: getattr(c, k) for k in SEL}, c.custom,
                         free_variables(c))
    assert rc == 0
    assert tuple(cols) == tuple(list(x) for x in c.wires_values())


def test_refusals_before_the_library(monkeypatch):
    import plonkathon_b200 as pb
    from plonkathon_b200 import solve as S

    def no_library():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(S, "lib", no_library)
    monkeypatch.setattr(S, "default_context", lambda: None)
    c = syn.build_circuit(4, seed=3)
    pk = {k: getattr(c, k) for k in SEL}
    args = (c.wire_L, c.wire_R, c.wire_O, pk)
    n = c.group_order
    bad = [
        (dict(inputs=(np.array([1, 1]), np.zeros((2, 32), np.uint8))), "two inputs name variable 1"),
        (dict(inputs={-2: 1}), r"outside \[0, 2\^32 - 2\]"),
        (dict(inputs={2**32 - 1: 1}), r"outside \[0, 2\^32 - 2\]"),
        (dict(inputs={0: R}), "not reduced below r"),
        (dict(inputs=(np.array([0]), np.full((1, 32), 255, np.uint8))), "not reduced below r"),
        (dict(inputs=(np.array([0]), np.zeros((2, 32), np.uint8))), r"\(1, 32\) uint8"),
        (dict(inputs=5), "dict id -> value"),
        (dict(inputs={}, n_constraints=n + 1), "n_constraints"),
        (dict(inputs={}, n_constraints=-1), "n_constraints"),
        (dict(inputs={}, group_order=12), "power of two"),
        (dict(inputs={}, limit=-1), "limit"),
    ]
    for kw, msg in bad:
        kw.setdefault("group_order", n)
        with pytest.raises(ValueError, match=msg):
            pb.solve_wires(*args, **kw)
    wl = np.array(c.wire_L)
    wl[3] = 2**32 - 1
    with pytest.raises(ValueError, match=r"wire_L\[3\]"):
        pb.solve_wires(wl, c.wire_R, c.wire_O, pk, {}, n)
    with pytest.raises(ValueError, match="wire_R must be a 1-D"):
        pb.solve_wires(c.wire_L, np.zeros((n, 2), np.int64), c.wire_O, pk, {}, n)
    with pytest.raises(ValueError, match="pk lacks QO"):
        pb.solve_wires(*args[:3], {k: v for k, v in pk.items() if k != "QO"}, {}, n)
    with pytest.raises(ValueError, match="QC must have"):
        pb.solve_wires(*args[:3], dict(pk, QC=[0] * 3), {}, n)


# ---- GPU -------------------------------------------------------------------------------------------------------------
def _circuit_kw(c):
    kw = {}
    if c.custom:
        kw["custom"] = syn.custom_arrays(c)
    if c.shuffle:
        kw["shuffle"] = syn.shuffle_arrays(c)
    if c.lookup:
        kw["lookup"] = syn.lookup_arrays(c)
    if c.lookups:
        kw["lookups"] = syn.lookups_arrays(c)
    return kw


def _tensor_ints(t):
    return _ints(t.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", PROGRAMS)
def test_gpu_reference_programs(name):
    import plonkathon_b200 as pb
    e, ids, n, m, sel, inputs = _program(name)
    entry, arr = load_circuit(name)
    sol = pb.solve_wires(ids[:, 0], ids[:, 1], ids[:, 2], sel, inputs, n, n_constraints=m)
    assert sol.ok, str(sol)
    for k, X in zip("ABC", (sol.A, sol.B, sol.C)):
        got = _ints(X)
        assert got[:m] == arr[k][:m] and not any(got[m:]), k
    setup = pb.Setup.from_file(os.path.join(GOLDEN, "powersOfTau28_hez_final_11.head.ptau"))
    pk = {k: arr[k] for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")}
    raw = pb.Prover.from_arrays(setup, n, pk).prove_arrays(sol.A, sol.B, sol.C, [int(x) for x in entry["public"]])
    assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"]


@pytest.mark.gpu
@pytest.mark.parametrize("log_n", [4, 8, 12])
@pytest.mark.parametrize("kind", KINDS)
def test_gpu_synthetic_every_kind(kind, log_n):
    import plonkathon_b200 as pb
    from plonkathon_b200.prover import proof_kind
    c = kind_circuit(kind, log_n)
    n = c.group_order
    kw = _circuit_kw(c)
    sol = pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, {k: getattr(c, k) for k in SEL}, free_variables(c), n,
                         n_constraints=c.n_constraints, custom=kw.get("custom", ()), device=True)
    assert sol.ok, str(sol)
    want = [_le(x) for x in c.wires_values()]
    for X, w in zip((sol.A, sol.B, sol.C), want):
        assert X.is_cuda and np.array_equal(X.cpu().numpy(), w)
    pk, A, B, C, public = syn.circuit_arrays(c)
    setup = pb.Setup.generate(TAU, n + 9)
    prover = pb.Prover.from_arrays(setup, n, pk, **kw)
    assert prover.check_arrays(sol.A, sol.B, sol.C, public).ok
    assert prover.prove_arrays(sol.A, sol.B, sol.C, public) == prover.prove_arrays(A, B, C, public)
    if n >= 16:  # zero knowledge with fixed blinders: the same bytes from either side
        k = proof_kind(next_row=prover.next_row, shuffle=bool(c.shuffle), lookup=bool(c.lookup or c.lookups))
        blinders = [(7919 * i + 13) % R for i in range(k.blinders)]
        {"pb200_prover_set_zk": prover.set_zk, "pb200_prover_set_zk_lookup": prover.set_zk_lookup,
         "pb200_prover_set_zk_shuffle": prover.set_zk_shuffle}[k.zk](True, blinders)
        assert prover.prove_arrays(sol.A, sol.B, sol.C, public) == prover.prove_arrays(A, B, C, public)


@pytest.mark.gpu
def test_gpu_golden_2p20_from_inputs_only():
    import json
    import plonkathon_b200 as pb
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    c = syn.build_circuit(20, seed=rec["seed"], n_public=2)
    n = c.group_order
    pk, _, _, _, public = syn.circuit_arrays(c)
    sol = pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, pk, free_variables(c), n, n_constraints=c.n_constraints,
                         device=True)
    assert sol.ok, str(sol)
    prover = pb.Prover.from_arrays(pb.Setup.generate(TAU, n), n, pk)
    rep = prover.check_arrays(sol.A, sol.B, sol.C, public)
    assert rep.ok, str(rep)
    assert prover.prove_arrays(sol.A, sol.B, sol.C, public).hex() == rec["proof_hex"]


def _chain(log_n, width, seed=5):
    """`width` independent chains of a + b and a * b rows, interleaved row by row; every row reads its chain's
    previous row (so with width 1 every row depends on the one before it)"""
    rng = np.random.default_rng(seed)
    n = 1 << log_n
    m = n
    L = np.empty(m, np.int64)
    Rw = np.empty(m, np.int64)
    O = np.arange(m, dtype=np.int64) + 2 * width
    last = np.arange(width, dtype=np.int64)  # chain k starts from inputs k and width + k
    other = np.arange(width, 2 * width, dtype=np.int64)
    for r in range(m):
        k = r % width
        L[r], Rw[r] = last[k], other[k]
        other[k] = last[k]
        last[k] = O[r]
    mul = rng.integers(0, 2, m).astype(bool)
    sel = {"QL": [0 if x else R - 1 for x in mul], "QR": [0 if x else R - 1 for x in mul],
           "QM": [R - 1 if x else 0 for x in mul], "QO": [1] * m, "QC": [0] * m}
    inputs = {v: int(rng.integers(1, 2**62)) for v in range(2 * width)}
    return L, Rw, O, sel, inputs, n


@pytest.mark.gpu
@pytest.mark.parametrize("width", [1, 4096])
def test_gpu_dependency_paths(width):
    import plonkathon_b200 as pb
    L, Rw, O, sel, inputs, n = _chain(16, width)
    sol = pb.solve_wires(L, Rw, O, sel, inputs, n)
    assert sol.ok, str(sol)
    ids = np.stack([L, Rw, O], axis=1)
    want, _, _ = restate(ids, n, n, sel, [], inputs)
    assert [_ints(X) for X in (sol.A, sol.B, sol.C)] == want


@pytest.mark.gpu
def test_gpu_errors_and_refusals(monkeypatch):
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    n = 64
    # rows: 0: v2 = v0 + v1; 1: v3 = v2 * v9 (v9 nowhere defined: unset, two cells); 2: v4 = v5 + v0 (v5 defined by
    # row 5: order); 3: v6 = v6 + v0 (reads itself: order); 4: v9 on O with QO = 0 (not defining); 5: v5 = v0 + v0
    L = [0, 2, 5, 6, 0, 0]
    Rw = [1, 9, 0, 0, 0, 0]
    O = [2, 3, 4, 6, 9, 5]
    one, neg = 1, R - 1
    sel = {"QL": [neg, 0, neg, neg, 0, neg] + [0] * (n - 6), "QR": [neg, 0, neg, neg, 0, neg] + [0] * (n - 6),
           "QM": [0, neg, 0, 0, 0, 0] + [0] * (n - 6), "QO": [one, one, one, one, 0, one] + [0] * (n - 6),
           "QC": [0] * n}
    inputs = {0: 3, 1: 4}
    sol = pb.solve_wires(L, Rw, O, sel, inputs, n, n_constraints=6, limit=16)
    assert not sol.ok and sol.A is None
    assert (sol.unset, sol.order) == (2, 2)
    assert sol.unset_cells == [3 * 1 + 1, 3 * 4 + 2]
    assert sol.order_cells == [(3 * 2 + 0, 5), (3 * 3 + 0, 3)]
    text = str(sol)
    assert "wires unsolved: 2 unset, 2 order" in text
    assert "unset: cell (row 1, R) variable 9 is neither an input nor defined by a row" in text
    assert "order: row 2 reads variable 5 (cell (2, L)), which row 5 defines" in text
    ids = np.full((n, 3), -1, np.int64)
    ids[:6] = np.stack([L, Rw, O], axis=1)
    _, unset, order = restate(ids, n, 6, sel, [], inputs)
    assert (unset, order) == (sol.unset_cells, sol.order_cells)
    short = pb.solve_wires(L, Rw, O, sel, inputs, n, n_constraints=6, limit=1)
    assert (short.unset, short.order, short.unset_cells, short.order_cells) == (2, 2, [4], [(6, 5)])
    assert "unset: 1 more" in str(short)

    # refusals inside the library name their fault and leave the context solving and proving
    vp = ctypes.c_void_p
    ctx = pb.default_context()
    ids6 = np.full((n, 3), -1, np.int64)
    ids6[:6] = np.stack([L, Rw, O], axis=1)
    sels = [_le(sel[k]) for k in SEL]
    sel_arr = (vp * 5)(*[s.ctypes.data for s in sels])
    out = [np.zeros((n, 32), np.uint8) for _ in range(3)]
    counts = (ctypes.c_uint64 * 2)()
    lists = (ctypes.c_uint32 * 3)()

    def call(ids_, in_ids, in_vals, log_n=6):
        in_ids = np.asarray(in_ids, np.int64)
        return _lib.lib().pb200_solve_wires(ctx.handle, ids_.ctypes.data_as(vp), log_n, 6, sel_arr, 0, b"\0",
                                            (vp * 1)(), len(in_ids), in_ids.ctypes.data_as(vp),
                                            in_vals.ctypes.data_as(vp), 1, counts, lists,
                                            (vp * 3)(*[o.ctypes.data for o in out]), 0)

    two = _le([3, 4])
    bad_ids = ids6.copy()
    bad_ids[4, 1] = -5
    assert call(bad_ids, [0, 1], two) == 1
    assert "at cell 13 (row 4, wire R)" in _lib.lib().pb200_last_error().decode()
    assert call(ids6, [1, 1], two) == 1
    assert "both name variable 1" in _lib.lib().pb200_last_error().decode()
    assert call(ids6, [0, 1], _le([3, R])) == 1
    assert "not reduced" in _lib.lib().pb200_last_error().decode()
    assert call(ids6, [0, 1], two, log_n=27) == 1
    assert "1 <= k <= 26" in _lib.lib().pb200_last_error().decode()
    monkeypatch.setenv("PB200_SOLVE_MAX_BYTES", "1000")
    assert call(ids6, [0, 1], two) == 1
    assert "needs" in _lib.lib().pb200_last_error().decode() and "1000 are free" in \
        _lib.lib().pb200_last_error().decode()
    monkeypatch.delenv("PB200_SOLVE_MAX_BYTES")
    test_gpu_reference_programs("prover_test")


@pytest.mark.gpu
def test_gpu_sharded_prover_refuses_device_tensors():
    import torch
    import plonkathon_b200 as pb
    from plonkathon_b200.parallel import ShardedProver
    p = ShardedProver.__new__(ShardedProver)
    p.group_order = 8
    p.ctx = pb.default_context()
    p._kind = pb.prover.KINDS[()]
    t = [torch.zeros((8, 32), dtype=torch.uint8, device="cuda") for _ in range(3)]
    with pytest.raises(ValueError, match="sharded prover"):
        p.prove_arrays(*t, [])


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("PB200_TEST_2P24") != "1", reason="opt-in: PB200_TEST_2P24=1")
def test_gpu_2p24_sliced_from_device_tensors():
    import plonkathon_b200 as pb
    from oracle import plonk_oracle as O  # noqa: F401
    c = syn.build_circuit(24, seed=7, n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    inputs = free_variables(c)
    sol = pb.solve_wires(c.wire_L, c.wire_R, c.wire_O, pk, inputs, n, n_constraints=c.n_constraints, device=True)
    assert sol.ok, str(sol)
    for X, H in zip((sol.A, sol.B, sol.C), (A, B, C)):
        assert hashlib.sha256(X.cpu().numpy().tobytes()).hexdigest() == hashlib.sha256(H.tobytes()).hexdigest()
    del c, A, B, C
    setup = pb.Setup.generate(TAU, n)
    prover = pb.Prover.from_arrays(setup, n, pk)
    assert prover.sliced
    raw = prover.prove_arrays(sol.A, sol.B, sol.C, public)
    del prover, sol
    vk = setup.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), pub)
    assert vk.verify_proof_unoptimized(n, pb.Proof.from_bytes(raw), pub)
