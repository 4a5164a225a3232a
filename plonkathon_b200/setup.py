"""Drop-in for the reference's ``setup.py``: ``Setup`` with ``from_file`` (setup.py:24-63),
``commit`` (setup.py:66-72) and ``verification_key`` (setup.py:75-77).  The SRS lives in HBM
(Montgomery form -- the same encoding the .ptau file uses on disk) together with the fixed-base
window table used by the MSM."""
from __future__ import annotations

import ctypes
from typing import Optional

from . import _lib
from .curve import G2, Scalar, _pt_bytes, _pt_from, g2_mul
from .field import CURVE_ORDER, FIELD_MODULUS, FQ, FQ2
from .custom_gates import is_next_row, split_terms
from .lookup import check_lookup, check_lookups, padded_table, to_le_rows
from .shuffle import check_shuffle
from .poly import Basis, Polynomial, _log2_exact
from .prover import _as_le_rows
from .verifier import VerificationKey  # noqa: F401  (re-exported: the reference's setup.py imports it too)

SETUP_FILE_G1_STARTPOS = 80  # setup.py:11
SETUP_FILE_POWERS_POS = 60  # setup.py:12
_G2_GEN_X_C0 = 10857046999023057135944570762232829481370756359578518086990519993285655852781
PTAU_SECTION_LAGRANGE_G1 = 12  # snarkjs binfile: [L_i(tau)]_1 for every domain size 2^p, block p at point offset 2^p - 1


def decode_ptau_coordinates(raw: bytes, factor: int) -> bytes:
    """.ptau coordinates (32-byte little-endian, multiplied by ``factor`` = 2^256 mod q) -> canonical little-endian."""
    finv = pow(factor, -1, FIELD_MODULUS)
    return b"".join((int.from_bytes(raw[i:i + 32], "little") * finv % FIELD_MODULUS).to_bytes(32, "little")
                    for i in range(0, len(raw) - 31, 32))


def ptau_sections(contents: bytes) -> dict:
    """Section table of a snarkjs binfile: {section id: (data offset, size)}.  Layout: b"ptau", u32 version,
    u32 section count, then per section u32 id, u64 size, data.  Sections cut off by a truncated file are left
    out (the reference's reader never looks at the table: it takes byte 60 and byte 80, setup.py:11-12,27)."""
    if len(contents) < 12 or contents[:4] != b"ptau":
        return {}
    count = int.from_bytes(contents[8:12], "little")
    out, pos = {}, 12
    for _ in range(count):
        if pos + 12 > len(contents):
            break
        sid = int.from_bytes(contents[pos:pos + 4], "little")
        size = int.from_bytes(contents[pos + 4:pos + 12], "little")
        if pos + 12 + size <= len(contents):
            out[sid] = (pos + 12, size)
        pos += 12 + size
    return out


PTAU_SECTION_HEADER, PTAU_SECTION_TAU_G1, PTAU_SECTION_TAU_G2 = 1, 2, 3


def ptau_layout(f) -> dict:
    """Section table of an open snarkjs binfile, read by seeking: {section id: (data offset, declared size, bytes
    present)}.  Follows ``ptau_sections``' layout, but keeps a section the file cuts off, with the bytes it has.  Raises
    ValueError for a wrong magic or a section header cut off."""
    f.seek(0, 2)
    file_size = f.tell()
    f.seek(0)
    head = f.read(12)
    if len(head) < 12 or head[:4] != b"ptau":
        raise ValueError("ptau: not a .ptau file (the magic 'ptau' is missing)")
    count = int.from_bytes(head[8:12], "little")
    out, pos = {}, 12
    for _ in range(count):
        if pos >= file_size:
            break
        f.seek(pos)
        sh = f.read(12)
        if len(sh) < 12:
            raise ValueError("ptau: the header of section %d is cut off at byte %d" % (len(out) + 1, pos))
        sid, size = int.from_bytes(sh[:4], "little"), int.from_bytes(sh[4:12], "little")
        out[sid] = (pos + 12, size, max(0, min(size, file_size - pos - 12)))
        pos += 12 + size
    return out


def _ptau_header(f, sections) -> int:
    """section 1: n8 = 32, q = BN254's q; returns the power p"""
    if PTAU_SECTION_HEADER not in sections:
        raise ValueError("ptau: section 1 (header) is missing")
    off, size, have = sections[PTAU_SECTION_HEADER]
    if have < 40 or have < size:
        raise ValueError("ptau: section 1 (header) is truncated")
    f.seek(off)
    h = f.read(40)
    n8 = int.from_bytes(h[:4], "little")
    if n8 != 32:
        raise ValueError("ptau: section 1 says n8 = %d, BN254 has 32-byte coordinates" % n8)
    if int.from_bytes(h[4:36], "little") != FIELD_MODULUS:
        raise ValueError("ptau: section 1 names a field modulus that is not BN254's q")
    return int.from_bytes(h[36:40], "little")


def _mont_to_int(raw: bytes) -> int:
    return int.from_bytes(raw, "little") * pow(2, -256, FIELD_MODULUS) % FIELD_MODULUS


class Setup:
    def __init__(self, powers_of_x, X2, ctx: Optional[_lib.Context] = None, precompute: bool = True):
        self._powers = list(powers_of_x)
        self._n = len(self._powers)
        self.X2 = X2
        self.tau = None
        self._lagrange = {}        # domain size -> SRS handle holding [L_i(tau)]_1
        self._lagrange_raw = None  # canonical x||y bytes of the .ptau Lagrange section (blocks of 2^p points)
        self._ptau_lagrange = None  # (file name, offset, bytes) of the .ptau Lagrange section (from_ptau)
        self._precompute = precompute
        self.ctx = ctx or _lib.default_context()
        raw = b"".join(_pt_bytes(p) for p in self._powers)
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().pb200_srs_create(self.ctx.handle, raw, self._n, 1 if precompute else 0,
                                               ctypes.byref(h)))
        self._srs = h

    @classmethod
    def generate(cls, tau: int, n: int, ctx: Optional[_lib.Context] = None, precompute: bool = True):
        """Structured test SRS [tau^i]G, i < n, generated on the GPU (the shipped .ptau stops at 2^11 powers,
        setup.py:27).  ``powers_of_x`` is materialised lazily; ``X2`` = [tau]_2 comes from the library's host G2
        arithmetic.  tau = 0 mod r raises ValueError: every point after the first would be the identity."""
        if tau % CURVE_ORDER == 0:
            raise ValueError("tau == 0 mod r: every SRS point after the first would be the identity")
        self = cls.__new__(cls)
        self._powers = None
        self._n = n
        self._lagrange = {}
        self._lagrange_raw = None
        self._ptau_lagrange = None
        self._precompute = precompute
        self.tau = tau % CURVE_ORDER
        self.X2 = g2_mul(G2, self.tau)
        self.ctx = ctx or _lib.default_context()
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().pb200_srs_generate(self.ctx.handle, self.tau.to_bytes(32, "little"), n,
                                                 1 if precompute else 0, ctypes.byref(h)))
        self._srs = h
        return self

    def export_points(self, first: int, count: int):
        buf = ctypes.create_string_buffer(64 * count)
        _lib.check(_lib.lib().pb200_srs_export(self.ctx.handle, self._srs, buf, first, count))
        raw = buf.raw
        return [(FQ(int.from_bytes(raw[64 * k:64 * k + 32], "little")),
                 FQ(int.from_bytes(raw[64 * k + 32:64 * k + 64], "little"))) for k in range(count)]

    def export_points_array(self, first: int, count: int):
        """the same points as a (count, 64) uint8 array (x || y little-endian), without building Python objects"""
        import numpy as np
        buf = np.empty((count, 64), dtype=np.uint8)
        _lib.check(_lib.lib().pb200_srs_export(self.ctx.handle, self._srs, buf.ctypes.data_as(ctypes.c_void_p), first, count))
        return buf

    @property
    def powers_of_x(self):
        if self._powers is None:
            self._powers = self.export_points(0, self._n)
        return self._powers

    def __del__(self):
        try:
            for h in getattr(self, "_lagrange", {}).values():
                if h:
                    _lib.lib().pb200_srs_destroy(h)
            self._lagrange = {}
            if getattr(self, "_srs", None):
                _lib.lib().pb200_srs_destroy(self._srs)
                self._srs = None
        except Exception:
            pass

    @classmethod
    def from_file(cls, filename, ctx=None, precompute=True):
        """setup.py:24-63 -- snarkjs .ptau: byte 60 = log2(#powers), G1 points from byte 80 as
        32-byte little-endian coordinates scaled by a constant recovered from the first point."""
        contents = open(filename, "rb").read()
        powers = 2 ** contents[SETUP_FILE_POWERS_POS]
        end = SETUP_FILE_G1_STARTPOS + 64 * powers
        values = [int.from_bytes(contents[i:i + 32], "little")
                  for i in range(SETUP_FILE_G1_STARTPOS, end, 32)]
        assert max(values) < FIELD_MODULUS
        factor = values[0] % FIELD_MODULUS  # first point is the generator, x == 1
        finv = pow(factor, -1, FIELD_MODULUS)
        values = [v * finv % FIELD_MODULUS for v in values]
        powers_of_x = [(FQ(values[2 * i]), FQ(values[2 * i + 1])) for i in range(powers)]
        target = (factor * _G2_GEN_X_C0 % FIELD_MODULUS).to_bytes(32, "little")
        pos = contents.find(target, end)
        assert pos >= 0, "G2 section not found"
        enc = contents[pos + 128: pos + 256]
        xv = [int.from_bytes(enc[i:i + 32], "little") * finv % FIELD_MODULUS for i in range(0, 128, 32)]
        X2 = (FQ2(xv[0:2]), FQ2(xv[2:4]))  # curve membership (setup.py:59) is checked by the library on first use
        self = cls(powers_of_x, X2, ctx=ctx, precompute=precompute)
        sec = ptau_sections(contents).get(PTAU_SECTION_LAGRANGE_G1)
        if sec is not None:
            self.load_lagrange_section(contents[sec[0]:sec[0] + sec[1]], factor)
        return self

    @classmethod
    def from_ptau(cls, filename, powers: Optional[int] = None, ctx=None, precompute: bool = True):
        """Ceremony SRS from a snarkjs .ptau, checked by the library (``pb200_srs_create_ptau``): every point reduced,
        on the curve and not the identity, point 0 the generator, [tau]_2 in G2, and the points successive powers of
        the tau behind [tau]_2.  Only the header, the section table and the needed byte ranges are read; the tauG1
        bytes go to the device as stored (Montgomery form), so no point becomes a Python object.

        ``powers``: how many tauG1 points to load; None takes 2^p (section 1's power, the count ``from_file`` takes),
        any count up to what section 2 holds (2^(p+1) - 1 in a ceremony file) is allowed.  A missing section, a wrong
        magic, a wrong q, or a truncated section 2 raises ValueError before any library call.  Section 3 (tauG2) may
        end after its second point, [tau]_2.  Section 12 (Lagrange blocks), if present, is read block by block in
        ``enable_lagrange``."""
        import numpy as np
        with open(filename, "rb") as f:
            sections = ptau_layout(f)
            p = _ptau_header(f, sections)
            if PTAU_SECTION_TAU_G1 not in sections:
                raise ValueError("ptau: section 2 (tauG1) is missing")
            g1_off, g1_size, g1_have = sections[PTAU_SECTION_TAU_G1]
            if g1_have < g1_size:
                raise ValueError("ptau: section 2 (tauG1) is truncated: %d of its %d bytes are in the file"
                                 % (g1_have, g1_size))
            if g1_size % 64:
                raise ValueError("ptau: section 2 (tauG1) is %d bytes, not a whole number of 64-byte points" % g1_size)
            held = g1_size // 64
            count = 2 ** p if powers is None else int(powers)
            if count < 1:
                raise ValueError("ptau: powers must be at least 1")
            if count > held:
                raise ValueError("Not enough powers in setup: %d asked for, the file's tauG1 section holds %d (power %d)"
                                 % (count, held, p))
            if PTAU_SECTION_TAU_G2 not in sections:
                raise ValueError("ptau: section 3 (tauG2) is missing")
            g2_off, _, g2_have = sections[PTAU_SECTION_TAU_G2]
            if g2_have < 256:
                raise ValueError("ptau: section 3 (tauG2) ends before its second point, [tau]_2")
            f.seek(g2_off + 128)
            tau_g2 = f.read(128)
        g1 = np.memmap(filename, dtype=np.uint8, mode="r", offset=g1_off, shape=(64 * count,))
        self = cls.__new__(cls)
        self._powers = None
        self._n = count
        self._lagrange = {}
        self._lagrange_raw = None
        self._ptau_lagrange = None
        self._precompute = precompute
        self.tau = None
        self.ctx = ctx or _lib.default_context()
        h = ctypes.c_void_p()
        _lib.check(_lib.lib().pb200_srs_create_ptau(self.ctx.handle, g1.ctypes.data_as(ctypes.c_void_p), count,
                                                    tau_g2, 1 if precompute else 0, ctypes.byref(h)))
        self._srs = h
        del g1
        c = [_mont_to_int(tau_g2[i:i + 32]) for i in range(0, 128, 32)]
        self.X2 = (FQ2(c[0:2]), FQ2(c[2:4]))
        sec = sections.get(PTAU_SECTION_LAGRANGE_G1)
        if sec is not None:
            self._ptau_lagrange = (filename, sec[0], sec[2])
        return self

    # ---- Lagrange-basis SRS (SURVEY 8(f) N4): commit = one MSM over the values, no inverse transform
    def load_lagrange_section(self, raw: bytes, factor: int = pow(2, 256, FIELD_MODULUS)):
        """``raw``: the data of .ptau section 12 (or a prefix of it): for p = 0, 1, 2, ... a block of 2^p points
        [L_i(tau)]_1 of the size-2^p domain, block p starting at point (2^p - 1); coordinates 32-byte little-endian,
        scaled by ``factor`` like the monomial section (setup.py:36-40)."""
        self._lagrange_raw = decode_ptau_coordinates(raw, factor)

    def enable_lagrange(self, n: int):
        """Make ``commit`` of n values use the Lagrange-basis points.  From a .ptau they come from section 12; for a
        generated SRS (known tau) they are computed on the device; a tau with tau^n = 1 (on the domain) raises
        ValueError, as every Lagrange point but one would be the identity."""
        if self._lagrange.get(n):
            return True
        h = ctypes.c_void_p()
        lag = getattr(self, "_ptau_lagrange", None)
        if lag is not None and 64 * (2 * n - 1) <= lag[2]:
            # block log2(n) of the .ptau's section 12, as stored, checked against the monomial points
            import numpy as np
            _log2_exact(n)
            block = np.memmap(lag[0], dtype=np.uint8, mode="r", offset=lag[1] + 64 * (n - 1), shape=(64 * n,))
            _lib.check(_lib.lib().pb200_srs_create_ptau_lagrange(
                self.ctx.handle, block.ctypes.data_as(ctypes.c_void_p), n, self._srs, 1 if self._precompute else 0,
                ctypes.byref(h)))
            del block
        elif self._lagrange_raw is not None and 64 * (2 * n - 1) <= len(self._lagrange_raw):
            block = self._lagrange_raw[64 * (n - 1):64 * (2 * n - 1)]
            _lib.check(_lib.lib().pb200_srs_create(self.ctx.handle, block, n, 1 if self._precompute else 0,
                                                   ctypes.byref(h)))
        elif getattr(self, "tau", None) is not None:
            if pow(self.tau, n, CURVE_ORDER) == 1:
                raise ValueError("tau^n == 1 mod r (tau is on the size-%d domain): every Lagrange point but one "
                                 "would be the identity" % n)
            _lib.check(_lib.lib().pb200_srs_generate_lagrange(self.ctx.handle, self.tau.to_bytes(32, "little"), n,
                                                              1 if self._precompute else 0, ctypes.byref(h)))
        else:
            return False
        self._lagrange[n] = h
        return True

    def disable_lagrange(self):
        for h in self._lagrange.values():
            _lib.lib().pb200_srs_destroy(h)
        self._lagrange = {}

    def commit(self, values: Polynomial):
        """setup.py:66-72."""
        assert values.basis == Basis.LAGRANGE
        n = len(values)
        if n > self._n:
            raise Exception("Not enough powers in setup")
        import torch
        d_vals = values._device(self.ctx)  # stays in HBM if it came out of a transform
        torch.cuda.current_stream(d_vals.device).synchronize()
        out = ctypes.create_string_buffer(64)
        ident = ctypes.c_int(0)
        lag = self._lagrange_handle(n)
        if lag is not None:
            _lib.check(_lib.lib().pb200_srs_commit_coeffs(
                self.ctx.handle, lag, ctypes.c_void_p(d_vals.data_ptr()), n, 0, out, ctypes.byref(ident)))
        else:
            _lib.check(_lib.lib().pb200_srs_commit_lagrange(
                self.ctx.handle, self._srs, ctypes.c_void_p(d_vals.data_ptr()), _log2_exact(n), out,
                ctypes.byref(ident)))
        return _pt_from(out.raw, ident.value)

    def _lagrange_handle(self, n: int):
        """SRS of the size-n Lagrange basis if there is one: .ptau blocks are picked up on first use, device-generated
        ones only after ``enable_lagrange(n)`` (they cost as much HBM as the monomial SRS)."""
        h = self._lagrange.get(n)
        if h is None and (self._lagrange_raw is not None or getattr(self, "_ptau_lagrange", None) is not None) \
                and self.enable_lagrange(n):
            h = self._lagrange[n]
        return h

    def verification_key_arrays(self, group_order: int, pk_arrays: dict, custom=(), lookup=None,
                                lookups=None, shuffle=None) -> VerificationKey:
        """``verification_key`` for circuits that exist only as arrays (``Prover.from_arrays``): QM..S3 as
        (n,32) uint8 little-endian Lagrange values in host memory.  ``custom``: the circuit's custom gate terms
        ``((i, j, l), column)`` as given to ``Prover.from_arrays``; each column is committed too.  ``lookup``:
        ``(q_K, (t1, t2, t3))`` as given to ``Prover.from_arrays``; the key gains [q_K], [t1], [t2], [t3] (the table
        padded to n rows), the identity for a constant-zero column.  ``lookups``: several tables as given to
        ``Prover.from_arrays``; the key gains [q_K], [t1], [t2], [t3], [Q_T], [t4] (the tables concatenated and padded).
        Not together with ``lookup``.  A custom term may have six exponents (i, j, l, i', j', l') and read the next
        row; the key then takes ``NextRowProof`` only.  Next-row terms do not combine with lookups (ValueError).
        ``shuffle``: ``(q_in, q_out)`` as given to ``Prover.from_arrays``; the key gains [q_in], [q_out] and takes
        ``ShuffleProof`` only (``NextRowShuffleProof`` with a next-row term).  Not together with lookups (ValueError)."""
        import numpy as np
        if lookup is not None and lookups is not None:
            raise ValueError("pass either lookup= (one table) or lookups= (several tables), not both")
        if shuffle is not None and (lookup is not None or lookups is not None):
            raise ValueError("shuffles do not combine with lookups")
        log_n = _log2_exact(group_order)
        exps, ccols = split_terms(custom, group_order)
        if (lookup is not None or lookups is not None) and any(is_next_row(e) for e in exps):
            raise ValueError("lookups do not combine with next-row custom gate terms")
        lk = check_lookup(lookup, group_order) if lookup is not None else None
        lks = check_lookups(lookups, group_order) if lookups is not None else None
        sh = check_shuffle(shuffle, group_order) if shuffle is not None else None

        def commit_host(col):
            col = np.ascontiguousarray(col).view(np.uint8).reshape(-1, 32)
            assert col.shape[0] == group_order
            out = ctypes.create_string_buffer(64)
            ident = ctypes.c_int(0)
            lag = self._lagrange_handle(group_order)
            if lag is not None:
                _lib.check(_lib.lib().pb200_srs_commit_coeffs_host(
                    self.ctx.handle, lag, col.ctypes.data_as(ctypes.c_void_p), group_order, out, ctypes.byref(ident)))
            else:
                _lib.check(_lib.lib().pb200_srs_commit_lagrange_host(
                    self.ctx.handle, self._srs, col.ctypes.data_as(ctypes.c_void_p), log_n, out, ctypes.byref(ident)))
            return _pt_from(out.raw, ident.value)

        pts = [commit_host(pk_arrays[k]) for k in ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")]
        terms = tuple((e, commit_host(_as_le_rows(col, group_order))) for e, col in zip(exps, ccols))
        lk_pts = ()
        if lk is not None:
            qk, cols, _rows = lk
            lk_pts = tuple(commit_host(to_le_rows(c)) for c in [qk] + padded_table(cols, group_order))
        if lks is not None:
            qk, qtag, cols, _rows = lks
            t1, t2, t3, t4 = padded_table(cols, group_order)
            lk_pts = tuple(commit_host(to_le_rows(c)) for c in (qk, t1, t2, t3, qtag, t4))
        sh_pts = tuple(commit_host(to_le_rows(q)) for q in sh) if sh is not None else ()
        return VerificationKey(group_order, *pts, self.X2, Scalar.root_of_unity(group_order), terms, lk_pts, sh_pts)

    def verification_key(self, pk) -> VerificationKey:
        """setup.py:75-77."""
        return VerificationKey(
            pk.group_order, self.commit(pk.QM), self.commit(pk.QL), self.commit(pk.QR), self.commit(pk.QO),
            self.commit(pk.QC), self.commit(pk.S1), self.commit(pk.S2), self.commit(pk.S3), self.X2,
            Scalar.root_of_unity(pk.group_order))
