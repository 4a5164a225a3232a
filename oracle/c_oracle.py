"""ORACLE / TEST INFRASTRUCTURE ONLY.  ctypes binding of oracle/c/libplonk_oracle_c.so (plonk_oracle.c): the
plain-C restatement of poly.py's fft/ifft and curve.py's ec_lincomb used for exact parity checks at sizes the
pure-Python oracle cannot reach in seconds, and the O(n) evaluations (Lagrange values or coefficients at one point)
that check a whole transform or commitment by one identity.  Built by `make -C oracle` (also from __graft_entry__.build())."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "c", "libplonk_oracle_c.so")
_lib = None


def lib():
    global _lib
    if _lib is None:
        src = os.path.join(_HERE, "c", "plonk_oracle.c")
        if not os.path.exists(_SO) or os.path.getmtime(src) > os.path.getmtime(_SO):
            subprocess.check_call(["make", "-s", "-C", _HERE])
        _lib = ctypes.CDLL(_SO)
    return _lib


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def fft(arr: np.ndarray, inverse: bool = False) -> np.ndarray:
    """arr: (n, 32) uint8 canonical little-endian -> same shape (poly.py:113-149)."""
    a = np.ascontiguousarray(arr, dtype=np.uint8)
    n = a.shape[0]
    out = np.empty_like(a)
    rc = lib().oc_fr_fft(_p(a), _p(out), n.bit_length() - 1, 1 if inverse else 0)
    assert rc == 0
    return out


def g1_lincomb(points: np.ndarray, scalars: np.ndarray):
    """points (n, 64) uint8, scalars (n, 32) uint8 -> (x, y) ints or None (curve.py:38-44)."""
    pts = np.ascontiguousarray(points, dtype=np.uint8)
    sc = np.ascontiguousarray(scalars, dtype=np.uint8)
    out = np.zeros(64, dtype=np.uint8)
    ident = ctypes.c_int(0)
    rc = lib().oc_g1_lincomb(_p(pts), _p(sc), ctypes.c_uint64(pts.shape[0]), _p(out), ctypes.byref(ident))
    if rc == 2:
        raise ValueError("max() arg is an empty sequence")
    assert rc == 0
    if ident.value:
        return None
    raw = out.tobytes()
    return int.from_bytes(raw[:32], "little"), int.from_bytes(raw[32:], "little")


def _rows(arr) -> np.ndarray:
    """field elements as (n, 32) uint8 rows, whatever the element width of the array (a view, not a cast)"""
    return np.ascontiguousarray(arr).view(np.uint8).reshape(-1, 32)


def _fr_bytes(x: int) -> np.ndarray:
    return np.frombuffer((int(x) % R_ORDER).to_bytes(32, "little"), dtype=np.uint8).copy()


def eval_lagrange(vals: np.ndarray, x: int) -> int:
    """value at x of the polynomial with Lagrange values `vals` on the n-th roots of unity (n a power of two, x off
    the domain)"""
    v = _rows(vals)
    n = v.shape[0]
    assert n and n & (n - 1) == 0, "the Lagrange basis needs a power-of-two domain"
    out = np.zeros(32, dtype=np.uint8)
    rc = lib().oc_fr_eval_lagrange(_p(v), n.bit_length() - 1, _p(_fr_bytes(x)), _p(out))
    assert rc == 0
    return int.from_bytes(out.tobytes(), "little")


def eval_coeffs(coeffs: np.ndarray, x: int) -> int:
    """sum_i coeffs[i] x^i for any length n (canonical scalars), by Horner"""
    c = _rows(coeffs)
    out = np.zeros(32, dtype=np.uint8)
    rc = lib().oc_fr_eval_coeffs(_p(c), ctypes.c_uint64(c.shape[0]), _p(_fr_bytes(x)), _p(out))
    assert rc == 0, "coefficient not reduced mod r" if rc == 2 else rc
    return int.from_bytes(out.tobytes(), "little")


def g1_powers(tau: int, n: int) -> np.ndarray:
    """[tau^i] G for i < n as an (n, 64) uint8 array (x || y canonical little-endian): the structured test SRS."""
    out = np.zeros((n, 64), dtype=np.uint8)
    rc = lib().oc_g1_powers(_p(_fr_bytes(tau)), ctypes.c_uint64(n), _p(out))
    assert rc == 0
    return out


R_ORDER = 21888242871839275222246405745257275088548364400416034343698204186575808495617
