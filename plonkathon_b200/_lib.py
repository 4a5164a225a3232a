"""ctypes binding of libplonk_b200.so (C ABI in include/plonk_b200.h).

There is no CPU fallback: if the shared library is missing, or no CUDA device is visible when a
context is requested, this module raises -- it never routes to another implementation."""
from __future__ import annotations

import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PB200_LIB") or os.path.join(_HERE, "libplonk_b200.so")  # PB200_LIB: tuning experiments

c_u8p = ctypes.POINTER(ctypes.c_uint8)


class PlonkB200Error(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise PlonkB200Error(
            "libplonk_b200.so is not built (%s); run `python -c 'import __graft_entry__ as g; g.build()'`"
            % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    V, I, U, U64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_uint64
    P = ctypes.POINTER
    sig = {
        "pb200_last_error": (ctypes.c_char_p, []),
        "pb200_version": (ctypes.c_char_p, []),
        "pb200_ctx_create": (I, [I, V, P(V)]),
        "pb200_ctx_destroy": (None, [V]),
        "pb200_ctx_sync": (I, [V]),
        "pb200_ctx_launches": (U64, [V]),
        "pb200_ctx_stream": (V, [V]),
        "pb200_ctx_timing": (I, [V, I]),
        "pb200_ctx_timing_read": (I, [V, I, P(ctypes.c_double), P(U64)]),
        "pb200_fr_to_mont": (I, [V, V, V, U64]),
        "pb200_fr_from_mont": (I, [V, V, V, U64]),
        "pb200_fr_ntt": (I, [V, V, V, U, I]),
        "pb200_fr_ntt_host": (I, [V, V, V, U, I]),
        "pb200_fr_ntt_decimated": (I, [V, V, V, U, I, U64, U64]),
        "pb200_fr_ntt_sharded": (I, [V, V, V, U, I]),
        "pb200_fr_vec_op": (I, [V, I, V, V, V, V, U64, U64]),
        "pb200_prover_read_vector": (I, [V, I, V]),
        "pb200_comm_unique_id": (I, [V]),
        "pb200_comm_init": (I, [V, V, I, I]),
        "pb200_comm_info": (I, [V, P(I), P(I), P(U64), P(U64)]),
        "pb200_srs_commit_coeffs_sharded": (I, [V, V, V, U64, I, V, P(I)]),
        "pb200_prover_create_sharded": (I, [V, V, U, V, P(V)]),
        "pb200_srs_commit_partial": (I, [V, V, V, U64, U64, U, U, I, V]),
        "pb200_srs_bucket_count": (I, [V, P(U)]),
        "pb200_g1_join_bucket_shards_host": (I, [V, U, U, U, V, P(I)]),
        "pb200_fr_coset_extend": (I, [V, V, V, U, V]),
        "pb200_fr_coset_extend_host": (I, [V, V, V, U, V]),
        "pb200_fr_coset_to_coeffs": (I, [V, V, V, U, V]),
        "pb200_fr_coset_to_coeffs_host": (I, [V, V, V, U, V]),
        "pb200_fr_barycentric_eval": (I, [V, V, U, V, V]),
        "pb200_fr_barycentric_eval_host": (I, [V, V, U, V, V]),
        "pb200_g1_msm": (I, [V, V, V, U64, V, P(I)]),
        "pb200_g1_msm_host": (I, [V, V, V, U64, V, P(I)]),
        "pb200_srs_create": (I, [V, V, U64, I, P(V)]),
        "pb200_srs_create_ptau": (I, [V, V, U64, V, I, P(V)]),
        "pb200_srs_create_ptau_lagrange": (I, [V, V, U64, V, I, P(V)]),
        "pb200_srs_ptau_stages": (None, [P(ctypes.c_double), I]),
        "pb200_srs_generate": (I, [V, V, U64, I, P(V)]),
        "pb200_srs_generate_lagrange": (I, [V, V, U64, I, P(V)]),
        "pb200_srs_export": (I, [V, V, V, U64, U64]),
        "pb200_srs_destroy": (None, [V]),
        "pb200_srs_size": (U64, [V]),
        "pb200_srs_commit_lagrange": (I, [V, V, V, U, V, P(I)]),
        "pb200_srs_commit_lagrange_host": (I, [V, V, V, U, V, P(I)]),
        "pb200_srs_commit_coeffs_host": (I, [V, V, V, U64, V, P(I)]),
        "pb200_srs_commit_coeffs": (I, [V, V, V, U64, I, V, P(I)]),
        "pb200_prover_create": (I, [V, V, U, V, P(V)]),
        "pb200_prover_create_custom": (I, [V, V, U, V, U, V, V, P(V)]),
        "pb200_prover_create_custom_sharded": (I, [V, V, U, V, U, V, V, P(V)]),
        "pb200_prover_destroy": (None, [V]),
        "pb200_prover_prove": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_prove_device": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_round1": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_round2": (I, [V, V, V, V]),
        "pb200_prover_round3": (I, [V, V, V, V]),
        "pb200_prover_round4": (I, [V, V, V]),
        "pb200_prover_round5": (I, [V, V, V]),
        "pb200_prover_serialize": (I, [V, V]),
        "pb200_prover_set_zk": (I, [V, I, V]),
        "pb200_prover_set_zk_lookup": (I, [V, I, V]),
        "pb200_prover_set_lookup": (I, [V, V, V, V, V, U64]),
        "pb200_prover_set_lookup_tagged": (I, [V, V, V, V, V, V, V, U64]),
        "pb200_prover_round_lookup": (I, [V, V, V]),
        "pb200_prover_round2_lookup": (I, [V, V, V, V, V, V]),
        "pb200_prover_round4_lookup": (I, [V, V, V]),
        "pb200_prover_prove_lookup": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_serialize_lookup": (I, [V, V]),
        "pb200_prover_create_custom_next_row": (I, [V, V, U, V, U, V, V, P(V)]),
        "pb200_prover_round4_next_row": (I, [V, V, V]),
        "pb200_prover_prove_next_row": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_serialize_next_row": (I, [V, V]),
        "pb200_prover_set_shuffle": (I, [V, V, V]),
        "pb200_prover_set_zk_shuffle": (I, [V, I, V]),
        "pb200_prover_round2_shuffle": (I, [V, V, V, V, V, V]),
        "pb200_prover_round4_shuffle": (I, [V, V, V]),
        "pb200_prover_round4_next_row_shuffle": (I, [V, V, V]),
        "pb200_prover_prove_shuffle": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_serialize_shuffle": (I, [V, V]),
        "pb200_prover_prove_next_row_shuffle": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_serialize_next_row_shuffle": (I, [V, V]),
        "pb200_g1_combine_partials_host": (I, [V, U, V, P(I)]),
        "pb200_transcript_create": (I, [V, ctypes.c_size_t, P(V)]),
        "pb200_transcript_destroy": (None, [V]),
        "pb200_transcript_append_message": (I, [V, V, ctypes.c_size_t, V, ctypes.c_size_t]),
        "pb200_transcript_challenge_bytes": (I, [V, V, ctypes.c_size_t, V, ctypes.c_size_t]),
        "pb200_transcript_get_and_append_challenge": (I, [V, V, ctypes.c_size_t, V]),
        "pb200_pairing_check": (I, [V, V, V, V, U, P(I)]),
        "pb200_g2_mul": (I, [V, V, V, P(I)]),
        "pb200_g2_add": (I, [V, I, V, I, V, P(I)]),
        "pb200_bench_modmul": (I, [V, I, U64, U, P(ctypes.c_float)]),
        "pb200_prover_sliced": (I, [V, P(I)]),
        "pb200_permutation": (I, [V, V, I, V]),
        "pb200_prover_check": (I, [V, V, V, V, V, U64, ctypes.c_uint32, V, V]),
        "pb200_prover_check_device": (I, [V, V, V, V, V, U64, ctypes.c_uint32, V, V]),
        "pb200_solve_wires": (I, [V, V, I, U64, V, U, V, V, U64, V, V, ctypes.c_uint32, V, V, V, I]),
        "pb200_solve_wires_lookup": (I, [V, V, I, U64, V, U, V, V, U64, V, V, V, V, V, V, V, V, U64,
                                         ctypes.c_uint32, V, V, V, V, I]),
        "pb200_solve_wires_shuffle": (I, [V, V, I, U64, V, U, V, V, U64, V, V, V, V, ctypes.c_uint32, V, V, V, I]),
        "pb200_solve_shuffle_stages": (None, [P(ctypes.c_double), I]),
        "pb200_prover_prove_device_lookup": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_prove_device_next_row": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_prove_device_shuffle": (I, [V, V, V, V, V, U64, V]),
        "pb200_prover_prove_device_next_row_shuffle": (I, [V, V, V, V, V, U64, V]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError here == ABI drift: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib, tuple(sig)


_lock = threading.Lock()
_lib = None
EXPORTS = ()


def lib():
    global _lib, EXPORTS
    with _lock:
        if _lib is None:
            _lib, EXPORTS = _load()
    return _lib


def check(rc):
    if rc != 0:
        raise PlonkB200Error(lib().pb200_last_error().decode())


class Context:
    """One per device (one process per GPU).  Owns the CUDA stream, NTT plans and scratch memory."""

    def __init__(self, device: int = 0, stream: int | None = None):
        h = ctypes.c_void_p()
        check(lib().pb200_ctx_create(device, ctypes.c_void_p(stream), ctypes.byref(h)))
        self.handle = h
        self.device = device

    def sync(self):
        check(lib().pb200_ctx_sync(self.handle))

    @property
    def launches(self) -> int:
        return int(lib().pb200_ctx_launches(self.handle))

    @property
    def stream(self) -> int:
        return int(lib().pb200_ctx_stream(self.handle) or 0)

    def close(self):
        if self.handle:
            lib().pb200_ctx_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default_ctx = None


def default_context() -> Context:
    """Context on LOCAL_RANK's device (one process per GPU), created on first use."""
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(int(os.environ.get("LOCAL_RANK", "0")))
    return _default_ctx
