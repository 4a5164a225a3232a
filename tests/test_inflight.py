"""Proofs in flight on one GPU: each context runs its MSM sort, stitch and upper reduction levels on a high-priority
stream of its own and joins them to its main stream with events.  These tests check that several contexts proving at
once, a context built on a caller's stream and the per-phase timers all still work."""
import ctypes
from concurrent.futures import ThreadPoolExecutor

import pytest

pytestmark = pytest.mark.gpu

TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
LOG_N = 16


@pytest.fixture(scope="module")
def env():
    import plonkathon_b200 as pb
    from plonkathon_b200 import synthetic as syn
    n = 1 << LOG_N
    setup = pb.Setup.generate(TAU, n)
    circuits = [syn.circuit_arrays(syn.build_circuit(LOG_N, seed=s, n_public=2)) for s in (21, 22, 23)]
    alone = [pb.Prover.from_arrays(setup, n, c[0]).prove_arrays(c[1], c[2], c[3], c[4]) for c in circuits]
    assert len(set(alone)) == 3
    return pb, setup, circuits, alone


def test_three_lanes_in_flight_match_one_lane(env):
    """three contexts proving at once from three host threads give, every time, the bytes one context gives alone.
    A missing join between a context's two streams would only fail here when the race it opens is lost, so this
    catches such a bug by chance; what it does check for certain is that contexts proving at once do not share state."""
    pb, setup, circuits, alone = env
    from plonkathon_b200 import _lib
    n = 1 << LOG_N
    lanes = [pb.Prover.from_arrays(setup, n, c[0], ctx=_lib.Context(0)) for c in circuits]

    def worker(i):
        c = circuits[i]
        return [lanes[i].prove_arrays(c[1], c[2], c[3], c[4]) for _ in range(4)]

    with ThreadPoolExecutor(3) as pool:
        got = list(pool.map(worker, range(3)))
    for i in range(3):
        assert got[i] == [alone[i]] * 4


def test_context_on_an_external_torch_stream(env):
    """a context on a caller's torch stream proves the same bytes, and its result is ready on that stream"""
    import torch
    pb, setup, circuits, alone = env
    from plonkathon_b200 import _lib
    n = 1 << LOG_N
    s = torch.cuda.Stream()
    ctx = _lib.Context(0, stream=s.cuda_stream)
    assert ctx.stream == s.cuda_stream
    c = circuits[1]
    prover = pb.Prover.from_arrays(setup, n, c[0], ctx=ctx)
    assert prover.prove_arrays(c[1], c[2], c[3], c[4]) == alone[1]
    s.synchronize()
    assert prover.prove_arrays(c[1], c[2], c[3], c[4]) == alone[1]


def test_timing_categories_count_every_msm_phase(env):
    """the per-phase event timers (bench.py's msm_ms_per_proof) still see one sort, one accumulation and one
    reduction per MSM call, with a positive duration, now that the phases run on two streams"""
    pb, setup, circuits, alone = env
    from plonkathon_b200 import _lib
    L = _lib.lib()
    n = 1 << LOG_N
    ctx = _lib.Context(0)
    c = circuits[0]
    prover = pb.Prover.from_arrays(setup, n, c[0], ctx=ctx)
    _lib.check(L.pb200_ctx_timing(ctx.handle, 1))
    try:
        assert prover.prove_arrays(c[1], c[2], c[3], c[4]) == alone[0]
        got = {}
        for cat in range(4):
            tot, cnt = ctypes.c_double(), ctypes.c_uint64()
            _lib.check(L.pb200_ctx_timing_read(ctx.handle, cat, ctypes.byref(tot), ctypes.byref(cnt)))
            got[cat] = (tot.value, cnt.value)
    finally:
        _lib.check(L.pb200_ctx_timing(ctx.handle, 0))
    accumulate, ntt, sort, reduce = got[0], got[1], got[2], got[3]
    assert sort[1] >= 1 and sort[1] == accumulate[1] == reduce[1], got
    assert ntt[1] >= 1, got
    assert all(v[0] > 0 for v in got.values()), got
