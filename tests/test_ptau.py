"""Ceremony SRS from a snarkjs .ptau (Setup.from_ptau -> pb200_srs_create_ptau / _lagrange): the tauG1 bytes go to
the device as stored and are checked there (reduced, on the curve, powers of the tau behind [tau]_2).

A small writer below makes snarkjs-format files (sections 1, 2, 3 and optionally 12, Montgomery coordinates) for the
test tau, from the oracle's C restatement or from the library's generated SRS.

CPU: the section parser on the shipped head of the Hermez 2^11 file, the writer's files round-trip, malformed headers
and truncations raise ValueError naming the fault.  GPU: the shipped ceremony points load and check (4095 of them) and
reproduce the golden proofs; a zero-knowledge proof at n = 2^11 verifies on them; a written 2^20 + 9 file equals the
generated SRS and reproduces the golden 2^20 proof; every refusal names its fault and leaves the context proving;
Lagrange blocks load and a corrupted one is refused.  PB200_TEST_PTAU_2P24=1 adds a 2^24 + 9 load and proof."""
import hashlib
import json
import os

import numpy as np
import pytest

from oracle import c_oracle as OC
from oracle import plonk_oracle as O
from plonkathon_b200 import synthetic as syn
from plonkathon_b200.setup import Setup, ptau_layout
from tests.golden_io import GOLDEN, PTAU_HEAD, ints, load_circuit, load_json

Q = 21888242871839275222246405745257275088696311157297823662689037894645226208583
R = O.R_MOD
RM = pow(2, 256, Q)  # Montgomery factor of the .ptau encoding
TAU = 0x1234567890ABCDEF1234567890ABCDEF1234567890ABCDEF
PK_KEYS = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")
G2_GEN = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
           11559732032986387107991004021392285783925812861821192530917403151452391805634),
          (8495653923123431417604973247489272438418190587263600148770280649306958101930,
           4082367875863433681332203403145435568316851327593401208105741076214120093531))


# ---- writer ---------------------------------------------------------------------------------------------------------
def to_mont(raw: bytes) -> bytes:
    """canonical 32-byte little-endian coordinates -> the .ptau's Montgomery encoding"""
    return b"".join((int.from_bytes(raw[i:i + 32], "little") * RM % Q).to_bytes(32, "little")
                    for i in range(0, len(raw), 32))


def from_mont(raw: bytes) -> bytes:
    inv = pow(RM, -1, Q)
    return b"".join((int.from_bytes(raw[i:i + 32], "little") * inv % Q).to_bytes(32, "little")
                    for i in range(0, len(raw), 32))


def g2_bytes(p) -> bytes:
    """((x0, x1), (y0, y1)) canonical ints -> 128 Montgomery bytes as section 3 stores a point"""
    return to_mont(b"".join(int(c).to_bytes(32, "little") for c in (p[0][0], p[0][1], p[1][0], p[1][1])))


def g2_ints(p):
    return tuple(tuple(c.n for c in coord.coeffs) for coord in p)


def write_ptau(path, power, g1_mont, tau_g2, lagrange_mont=None):
    """snarkjs binfile: sections 1 (n8, q, power, ceremony power), 2 (tauG1), 3 (tauG2: G2 then [tau]_2) and, if
    given, 12 (Lagrange blocks).  g1_mont: bytes or a list of byte chunks, Montgomery x || y per point."""
    chunks = [g1_mont] if isinstance(g1_mont, (bytes, bytearray)) else list(g1_mont)
    g1_size = sum(len(c) for c in chunks)
    g2 = g2_bytes(G2_GEN) + tau_g2
    header = (32).to_bytes(4, "little") + Q.to_bytes(32, "little") + power.to_bytes(4, "little") * 2
    with open(path, "wb") as f:
        f.write(b"ptau" + (1).to_bytes(4, "little") + (4 if lagrange_mont is not None else 3).to_bytes(4, "little"))
        f.write((1).to_bytes(4, "little") + len(header).to_bytes(8, "little") + header)
        f.write((2).to_bytes(4, "little") + g1_size.to_bytes(8, "little"))
        for c in chunks:
            f.write(c)
        f.write((3).to_bytes(4, "little") + len(g2).to_bytes(8, "little") + g2)
        if lagrange_mont is not None:
            f.write((12).to_bytes(4, "little") + len(lagrange_mont).to_bytes(8, "little") + lagrange_mont)


def oracle_powers_mont(n, tau=TAU) -> bytes:
    return to_mont(OC.g1_powers(tau, n).tobytes())


def _read(path, off, size):
    with open(path, "rb") as f:
        f.seek(off)
        return f.read(size)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_parser_on_the_shipped_head_fixture():
    with open(PTAU_HEAD, "rb") as f:
        sec = ptau_layout(f)
    assert sec[1] == (24, 44, 44)
    assert sec[2] == (80, 4095 * 64, 4095 * 64)  # 2^(p+1) - 1 points, all present
    off, size, have = sec[3]
    assert size == 2048 * 128 and have == 256  # tauG2 cut off after [tau]_2
    head = _read(PTAU_HEAD, 24, 44)
    assert int.from_bytes(head[:4], "little") == 32 and int.from_bytes(head[4:36], "little") == Q
    assert int.from_bytes(head[36:40], "little") == 11
    # point 0 decodes to the generator, and the file's points are the ones the reference reader takes
    g1 = _read(PTAU_HEAD, 80, 64 * 4)
    assert from_mont(g1[:64]) == (1).to_bytes(32, "little") + (2).to_bytes(32, "little")
    osetup = O.Setup.from_file(PTAU_HEAD)
    dec = from_mont(g1)
    assert [(int.from_bytes(dec[64 * i:64 * i + 32], "little"), int.from_bytes(dec[64 * i + 32:64 * i + 64], "little"))
            for i in range(4)] == [tuple(p) for p in osetup.powers_of_x[:4]]
    assert from_mont(_read(PTAU_HEAD, off, 128)) == b"".join(c.to_bytes(32, "little") for c in
                                                            (G2_GEN[0][0], G2_GEN[0][1], G2_GEN[1][0], G2_GEN[1][1]))


def test_writer_round_trips(tmp_path):
    import plonkathon_b200 as pb
    n = 40
    g1 = oracle_powers_mont(n)
    x2 = g2_ints(pb.g2_mul(pb.G2, TAU))
    lag = oracle_powers_mont(7, tau=5)  # stand-in bytes: the parser does not look inside section 12
    path = str(tmp_path / "t.ptau")
    write_ptau(path, 5, g1, g2_bytes(x2), lagrange_mont=lag)
    with open(path, "rb") as f:
        sec = ptau_layout(f)
    assert sorted(sec) == [1, 2, 3, 12]
    assert sec[2] == (80, 64 * n, 64 * n)
    assert _read(path, 80, 64 * n) == g1
    assert from_mont(_read(path, 80, 64 * n)) == OC.g1_powers(TAU, n).tobytes()
    off = sec[3][0]
    assert from_mont(_read(path, off + 128, 128)) == b"".join(c.to_bytes(32, "little") for c in
                                                             (x2[0][0], x2[0][1], x2[1][0], x2[1][1]))
    assert _read(path, sec[12][0], sec[12][1]) == lag
    # the reference's reader takes the same 2^5 points from a written file
    osetup = O.Setup.from_file(path)
    assert [tuple(p) for p in osetup.powers_of_x] == [
        (int.from_bytes(r[:32], "little"), int.from_bytes(r[32:], "little")) for r in OC.g1_powers(TAU, 32)]


def _malformed(tmp_path, name, data):
    p = str(tmp_path / name)
    with open(p, "wb") as f:
        f.write(data)
    return p


def test_malformed_files_raise_before_any_library_call(tmp_path):
    import plonkathon_b200 as pb
    good = str(tmp_path / "good.ptau")
    write_ptau(good, 4, oracle_powers_mont(31), g2_bytes(g2_ints(pb.g2_mul(pb.G2, TAU))))
    data = open(good, "rb").read()
    cases = [
        ("magic", b"ptaX" + data[4:], "magic"),
        ("empty", b"", "magic"),
        ("n8", data[:24] + (48).to_bytes(4, "little") + data[28:], "n8 = 48"),
        ("q", data[:28] + (Q + 2).to_bytes(32, "little") + data[60:], "not BN254's q"),
        ("cut_g1", data[:80 + 64 * 20], "section 2 .*truncated"),
        ("cut_header", data[:70], "header of section 2 is cut off"),
        ("cut_g2", data[:len(data) - 200], "section 3 .*second point"),
        ("no_g2", data[:12 - 4] + (2).to_bytes(4, "little") + data[12:80 + 64 * 31], "section 3 .*missing"),
        ("odd_g1", data[:72] + (64 * 31 - 1).to_bytes(8, "little") + data[80:], "not a whole number"),
    ]
    for name, blob, msg in cases:
        with pytest.raises(ValueError, match=msg):
            Setup.from_ptau(_malformed(tmp_path, name, blob))
    with pytest.raises(ValueError, match="Not enough powers in setup.*32 asked for.*holds 31"):
        Setup.from_ptau(good, powers=32)
    with pytest.raises(ValueError, match="Not enough powers in setup.*asked for.*holds 31"):
        Setup.from_ptau(_malformed(tmp_path, "p5", data[:60] + (5).to_bytes(4, "little") + data[64:]))


def _twist_point_outside_g2():
    """a point on y^2 = x^3 + 3/(9+u) that is not in G2 (the twist's cofactor is about q, so almost every point)"""
    def mul(a, b):
        return ((a[0] * b[0] - a[1] * b[1]) % Q, (a[0] * b[1] + a[1] * b[0]) % Q)

    def pw(a, e):
        r = (1, 0)
        while e:
            if e & 1:
                r = mul(r, a)
            a, e = mul(a, a), e >> 1
        return r

    inv = pow(82, -1, Q)  # 1/(9+u) = (9-u)/82
    b = (3 * 9 * inv % Q, -3 * inv % Q)
    x = (1, 0)
    while True:
        rhs = mul(mul(x, x), x)
        rhs = ((rhs[0] + b[0]) % Q, (rhs[1] + b[1]) % Q)
        a1 = pw(rhs, (Q - 3) // 4)  # q = 3 mod 4: the square root of Adj and Rodriguez-Henriquez, Algorithm 9
        alpha = mul(mul(a1, a1), rhs)
        x0 = mul(a1, rhs)
        if alpha == (Q - 1, 0):
            y = mul((0, 1), x0)
        else:
            y = mul(pw(((1 + alpha[0]) % Q, alpha[1]), (Q - 1) // 2), x0)
        if mul(y, y) == rhs:
            return x, y
        x = (x[0] + 1, 0)


def test_twist_point_outside_g2_is_refused_by_the_host_check():
    """the point the refusal test uses lies on the twist (the library's G2 loader checks that) and r P != O"""
    import ctypes
    from plonkathon_b200 import _lib

    def times_r(p):
        out, ident = ctypes.create_string_buffer(128), ctypes.c_int(0)
        raw = b"".join(int(c).to_bytes(32, "little") for c in (p[0][0], p[0][1], p[1][0], p[1][1]))
        _lib.check(_lib.lib().pb200_g2_mul(raw, R.to_bytes(32, "little"), out, ctypes.byref(ident)))
        return ident.value

    assert times_r(_twist_point_outside_g2()) == 0
    assert times_r(G2_GEN) == 1


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _export(setup, first=0, count=None):
    return setup.export_points_array(first, setup._n if count is None else count)


@pytest.mark.gpu
def test_gpu_head_fixture_matches_from_file_and_reproduces_golden_proofs():
    import plonkathon_b200 as pb
    ref = pb.Setup.from_file(PTAU_HEAD)
    s = pb.Setup.from_ptau(PTAU_HEAD, powers=2048)
    assert s._powers is None and s._n == 2048
    assert _export(s).tobytes() == _export(ref).tobytes()
    assert g2_ints(s.X2) == g2_ints(ref.X2)
    g = load_json("circuits.json")
    c = s.commit(pb.Polynomial([pb.Scalar(v) for v in ints(g["commit_kat"]["lagrange"])], pb.Basis.LAGRANGE))
    assert (c[0].n, c[1].n) == (16120260411117808045030798560855586501988622612038310041007562782458075125622,
                                3125847109934958347271782137825877642397632921923926105820408033549219695465)
    for name in ("prover_test", "factorization", "poseidon"):
        entry, arr = load_circuit(name)
        prover = pb.Prover.from_arrays(s, entry["n"], {k: arr[k] for k in PK_KEYS})
        raw = prover.prove_arrays(arr["A"], arr["B"], arr["C"], ints(entry["public"]))
        assert hashlib.sha256(raw).hexdigest() == entry["proof_sha256"], name
    # the default count is 2^p, what from_file takes
    assert pb.Setup.from_ptau(PTAU_HEAD, precompute=False)._n == 2048


@pytest.mark.gpu
def test_gpu_all_4095_ceremony_points_and_a_zero_knowledge_proof_at_2p11():
    import plonkathon_b200 as pb
    s = pb.Setup.from_ptau(PTAU_HEAD, powers=4095)
    ref = pb.Setup.from_file(PTAU_HEAD)
    assert _export(s, 0, 2048).tobytes() == _export(ref).tobytes()
    assert from_mont(_read(PTAU_HEAD, 80 + 64 * 2048, 64 * 2047)) == _export(s, 2048, 2047).tobytes()
    c = syn.build_circuit(11, seed=211, n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    prover = pb.Prover.from_arrays(s, n, pk)
    prover.set_zk(True)  # n + 6 = 2054 powers: more than from_file's 2048
    raw = prover.prove_arrays(A, B, C, public)
    vk = s.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    pf = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(n, pf, pub) and vk.verify_proof_unoptimized(n, pf, pub)
    assert not vk.verify_proof(n, pf, [pub[0] + 1] + pub[1:])
    assert not vk.verify_proof_unoptimized(n, pf, [pub[0] + 1] + pub[1:])


def _generated_file(pb, path, count, power):
    """a .ptau of `count` points for TAU from the library's generated SRS; returns that SRS"""
    gen = pb.Setup.generate(TAU, count)
    arr = gen.export_points_array(0, count)
    step = 1 << 18
    chunks = [to_mont(arr[i:i + step].tobytes()) for i in range(0, count, step)]
    write_ptau(path, power, chunks, g2_bytes(g2_ints(gen.X2)))
    return gen


@pytest.mark.gpu
def test_gpu_written_2p20_file_equals_generated_srs_and_reproduces_golden_proof(tmp_path):
    import plonkathon_b200 as pb
    count = (1 << 20) + 9
    path = str(tmp_path / "p20.ptau")
    gen = _generated_file(pb, path, count, 20)
    s = pb.Setup.from_ptau(path, powers=count)
    assert hashlib.sha256(_export(s).tobytes()).hexdigest() == hashlib.sha256(_export(gen).tobytes()).hexdigest()
    assert g2_ints(s.X2) == g2_ints(gen.X2)
    del gen
    rec = json.load(open(os.path.join(GOLDEN, "proof_2p20.json")))
    c = syn.build_circuit(rec["log_n"], seed=rec["seed"], n_public=rec["n_public"])
    pk, A, B, C, public = syn.circuit_arrays(c)
    raw = pb.Prover.from_arrays(s, c.group_order, pk).prove_arrays(A, B, C, public)
    assert raw.hex() == rec["proof_hex"], "proof on the loaded .ptau differs from the golden 2^20 proof"


@pytest.mark.gpu
def test_gpu_refusals_name_the_fault_and_leave_the_context_proving(tmp_path):
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    n, k = 4096, 2345
    g1 = bytearray(oracle_powers_mont(n))
    x2 = g2_bytes(g2_ints(pb.g2_mul(pb.G2, TAU)))
    good_path = str(tmp_path / "good.ptau")
    write_ptau(good_path, 12, bytes(g1), x2)
    good = pb.Setup.from_ptau(good_path, powers=n)
    probe = pb.Polynomial([pb.Scalar(v) for v in range(1, 65)], pb.Basis.LAGRANGE)
    expect = good.commit(probe)

    def point(i):
        return g1[64 * i:64 * i + 64]

    def with_point(i, raw):
        b = bytearray(g1)
        b[64 * i:64 * i + 64] = raw
        return bytes(b)

    x_k = int.from_bytes(point(k)[:32], "little")
    y_k = int.from_bytes(point(k)[32:], "little")
    double = OC.g1_lincomb(OC.g1_powers(TAU, n)[k:k + 1], np.frombuffer((2).to_bytes(32, "little"), np.uint8)[None])
    tx, ty = _twist_point_outside_g2()
    x2_int = g2_ints(pb.g2_mul(pb.G2, TAU))
    cases = [
        ("range", with_point(k, (x_k + Q).to_bytes(32, "little") + point(k)[32:]), x2,
         "ptau: tauG1 point %d has a coordinate that is not below q" % k),
        ("curve", with_point(k, point(k)[:32] + ((y_k + 1) % Q).to_bytes(32, "little")), x2,
         "ptau: tauG1 point %d is not on the curve" % k),
        ("identity", with_point(k, bytes(64)), x2, "ptau: tauG1 point %d is the identity" % k),
        ("power", with_point(k, to_mont(double[0].to_bytes(32, "little") + double[1].to_bytes(32, "little"))), x2,
         r"ptau: the tauG1 powers are not consistent with \[tau\]_2"),
        ("generator", with_point(0, point(1)), x2, r"ptau: tauG1 point 0 is not the generator \(1, 2\)"),
        ("wrong_tau", bytes(g1), g2_bytes(g2_ints(pb.g2_mul(pb.G2, TAU + 1))),
         r"ptau: the tauG1 powers are not consistent with \[tau\]_2"),
        ("twist", bytes(g1), g2_bytes((x2_int[0], ((x2_int[1][0] + 1) % Q, x2_int[1][1]))),
         r"ptau: \[tau\]_2 is not on the twist curve"),
        ("g2", bytes(g1), g2_bytes((tx, ty)), r"ptau: \[tau\]_2 is not in G2"),
    ]
    for name, blob, tg2, msg in cases:
        path = str(tmp_path / (name + ".ptau"))
        write_ptau(path, 12, blob, tg2)
        for pre in (True, False):
            with pytest.raises(_lib.PlonkB200Error, match=msg):
                pb.Setup.from_ptau(path, powers=n, precompute=pre)
        assert good.commit(probe) == expect, name  # the context is usable after the refusal
    with pytest.raises(ValueError, match="Not enough powers in setup.*4097 asked for.*holds 4096"):
        pb.Setup.from_ptau(good_path, powers=n + 1)
    # and proves after all of them
    c = syn.build_circuit(10, seed=77, n_public=2)
    pk, A, B, C, public = syn.circuit_arrays(c)
    raw = pb.Prover.from_arrays(good, c.group_order, pk).prove_arrays(A, B, C, public)
    vk = good.verification_key_arrays(c.group_order, pk)
    pub = [int(x) for x in public]
    pf = pb.Proof.from_bytes(raw)
    assert vk.verify_proof(c.group_order, pf, pub) and vk.verify_proof_unoptimized(c.group_order, pf, pub)


def _lagrange_blocks(pb, gen, top):
    """section 12 of a file for the generated SRS: blocks 2^0 .. 2^top of [L_i(tau)], Montgomery"""
    import ctypes
    from plonkathon_b200 import _lib
    out = [to_mont((1).to_bytes(32, "little") + (2).to_bytes(32, "little"))]  # L_0 = 1 on the one-point domain
    for p in range(1, top + 1):
        m = 1 << p
        assert gen.enable_lagrange(m)
        buf = np.empty((m, 64), dtype=np.uint8)
        _lib.check(_lib.lib().pb200_srs_export(gen.ctx.handle, gen._lagrange[m], buf.ctypes.data_as(ctypes.c_void_p),
                                               0, m))
        out.append(to_mont(buf.tobytes()))
    gen.disable_lagrange()
    return out


@pytest.mark.gpu
def test_gpu_lagrange_blocks_load_checked_and_corrupt_ones_are_refused(tmp_path):
    import ctypes
    import plonkathon_b200 as pb
    from plonkathon_b200 import _lib
    n = 4096
    gen = pb.Setup.generate(TAU, n)
    g1 = to_mont(gen.export_points_array(0, n).tobytes())
    x2 = g2_bytes(g2_ints(gen.X2))
    blocks = _lagrange_blocks(pb, gen, 12)
    path = str(tmp_path / "lag.ptau")
    write_ptau(path, 12, g1, x2, lagrange_mont=b"".join(blocks))
    s = pb.Setup.from_ptau(path, powers=n)
    assert s._ptau_lagrange is not None and s._lagrange_raw is None
    assert s.enable_lagrange(n) and s.enable_lagrange(16)
    want = np.empty((n, 64), dtype=np.uint8)
    gen.enable_lagrange(n)
    _lib.check(_lib.lib().pb200_srs_export(gen.ctx.handle, gen._lagrange[n], want.ctypes.data_as(ctypes.c_void_p), 0, n))
    got = np.empty((n, 64), dtype=np.uint8)
    _lib.check(_lib.lib().pb200_srs_export(s.ctx.handle, s._lagrange[n], got.ctypes.data_as(ctypes.c_void_p), 0, n))
    assert got.tobytes() == want.tobytes()
    # commitments through the block equal the monomial path's
    vals = [pb.Scalar(v * 7 + 1) for v in range(n)]
    via_block = s.commit(pb.Polynomial(vals, pb.Basis.LAGRANGE))
    s.disable_lagrange()
    s._ptau_lagrange = None
    assert s.commit(pb.Polynomial(vals, pb.Basis.LAGRANGE)) == via_block
    # one Lagrange point replaced by another point of the curve: only the commitment check can see it
    j = 1234
    bad = bytearray(blocks[12])
    bad[64 * j:64 * j + 64] = blocks[12][64 * (j + 1):64 * (j + 2)]
    top = b"".join(blocks[:12])
    for name, blk, msg in (
            ("swap", bytes(bad), "ptau: the Lagrange block of size 4096 is not consistent with the tauG1 powers"),
            ("curve", bytes(blocks[12][:64 * j + 32]) + bytes(32) + blocks[12][64 * j + 64:],
             "ptau: Lagrange point %d (is not on the curve|is the identity)" % j)):
        p = str(tmp_path / ("lag_" + name + ".ptau"))
        write_ptau(p, 12, g1, x2, lagrange_mont=top + blk)
        t = pb.Setup.from_ptau(p, powers=n)
        with pytest.raises(_lib.PlonkB200Error, match=msg):
            t.enable_lagrange(n)
        assert t.enable_lagrange(2048)  # smaller blocks are intact


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get("PB200_TEST_PTAU_2P24") != "1", reason="set PB200_TEST_PTAU_2P24=1 (writes 1 GiB)")
def test_gpu_2p24_file_loads_and_proves(tmp_path):
    import plonkathon_b200 as pb
    count = (1 << 24) + 9
    path = str(tmp_path / "p24.ptau")
    gen = _generated_file(pb, path, count, 24)
    del gen
    s = pb.Setup.from_ptau(path, powers=count)
    c = syn.build_circuit(24, seed=5, n_public=2)
    n = c.group_order
    pk, A, B, C, public = syn.circuit_arrays(c)
    raw = pb.Prover.from_arrays(s, n, pk).prove_arrays(A, B, C, public)
    vk = s.verification_key_arrays(n, pk)
    pub = [int(x) for x in public]
    assert vk.verify_proof(n, pb.Proof.from_bytes(raw), pub)
