"""CPU: the C restatement (oracle/c/plonk_oracle.c) against the pinned Python oracle and the golden vectors."""
import random

import numpy as np

from oracle import c_oracle as C
from oracle import plonk_oracle as O
from tests.golden_io import PTAU_HEAD, ints, load_json, pt


def le(ints_):
    return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in ints_), dtype=np.uint8).reshape(-1, 32).copy()


def un(arr):
    raw = arr.tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


def test_c_fft_matches_golden_and_python_oracle():
    for c in load_json("fft_vectors.json")["cases"]:
        v = ints(c["input"])
        assert un(C.fft(le(v))) == ints(c["fft"])
        assert un(C.fft(le(v), True)) == ints(c["ifft"])
    rng = random.Random(2)
    v = [rng.randrange(O.R_MOD) for _ in range(1 << 12)]
    assert un(C.fft(le(v))) == O.fft(v)


def test_c_lincomb_matches_golden_and_python_oracle():
    for c in load_json("lincomb_vectors.json")["cases"]:
        pairs = [(pt(p), int(s) % O.R_MOD) for p, s in zip(c["points"], c["scalars"]) if p is not None]
        if not pairs:
            continue
        pts = np.frombuffer(b"".join(p[0].to_bytes(32, "little") + p[1].to_bytes(32, "little") for p, _ in pairs),
                            dtype=np.uint8).reshape(-1, 64)
        assert C.g1_lincomb(pts, le([s for _, s in pairs])) == O.ec_lincomb_naive(pairs), c["name"]
    s = O.Setup.from_file(PTAU_HEAD)
    rng = random.Random(3)
    n = 700
    sc = [rng.randrange(O.R_MOD) for _ in range(n)]
    pts = np.frombuffer(b"".join(p[0].to_bytes(32, "little") + p[1].to_bytes(32, "little") for p in s.powers_of_x[:n]),
                        dtype=np.uint8).reshape(-1, 64)
    assert C.g1_lincomb(pts, le(sc)) == O.ec_lincomb(list(zip(s.powers_of_x[:n], sc)))


def test_c_eval_lagrange():
    rng = random.Random(4)
    v = [rng.randrange(O.R_MOD) for _ in range(256)]
    v[3] = 0
    x = rng.randrange(O.R_MOD)
    assert C.eval_lagrange(le(v), x) == O.eval_lagrange_at(v, x) == O.barycentric_eval(v, x)


def _horner(c, x):
    acc = 0
    for v in reversed(c):
        acc = (acc * x + v) % O.R_MOD
    return acc


def test_c_eval_coeffs_against_python_ints():
    """oc_fr_eval_coeffs (Horner) against Python ints: lengths 1, 2, 3, powers of two and 2^k + 3, zero and r - 1
    coefficients, x = 0, 1, r - 1 and random points"""
    rng = random.Random(5)
    R = O.R_MOD
    xs = [0, 1, R - 1, 2, rng.randrange(R), rng.randrange(R)]
    for n in (1, 2, 3, 4, 7, 8, 11, 64, 67, 1024, 1027):
        cases = {
            "random": [rng.randrange(R) for _ in range(n)],
            "zeros": [0] * n,
            "r-1": [R - 1] * n,
            "mixed": [rng.choice([0, 1, R - 1, rng.randrange(R)]) for _ in range(n)],
        }
        for name, c in cases.items():
            arr = le(c)
            for x in xs:
                want = _horner(c, x)
                assert C.eval_coeffs(arr, x) == want, (n, name, x)
    # x = 0 picks c_0, x = 1 sums, x = r - 1 alternates
    c = [rng.randrange(R) for _ in range(9)]
    assert C.eval_coeffs(le(c), 0) == c[0]
    assert C.eval_coeffs(le(c), 1) == sum(c) % R
    assert C.eval_coeffs(le(c), R - 1) == sum(v if i % 2 == 0 else -v for i, v in enumerate(c)) % R
    # the same bytes viewed as uint32 limbs give the same value; an empty vector is the zero polynomial
    assert C.eval_coeffs(le(c).view(np.uint32), 12345) == _horner(c, 12345)
    assert C.eval_coeffs(np.zeros((0, 32), dtype=np.uint8), 7) == 0


def test_c_eval_coeffs_agrees_with_eval_lagrange_through_the_fft():
    """the identity the GPU transform tests rest on: eval_lagrange(FFT(c), z) == eval_coeffs(c, z), and
    eval_coeffs(IFFT(v), z) == eval_lagrange(v, z), with the C FFT at 2^10"""
    rng = random.Random(6)
    c = le([rng.randrange(O.R_MOD) for _ in range(1 << 10)])
    z = rng.randrange(O.R_MOD)
    assert C.eval_lagrange(C.fft(c), z) == C.eval_coeffs(c, z)
    assert C.eval_coeffs(C.fft(c, True), z) == C.eval_lagrange(c, z)
    assert C.eval_coeffs(C.fft(c, True), z) != C.eval_lagrange(c, (z + 1) % O.R_MOD)
