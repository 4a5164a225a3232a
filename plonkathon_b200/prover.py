"""Drop-in for the reference's ``prover.py``: ``Proof`` (prover.py:11-35) and ``Prover`` with
``prove`` and ``round_1..5`` (prover.py:39-306).  The rounds run on the GPU through the C ABI
(csrc/prover.cu); vectors stay device-resident between rounds and only the 9 points + 6 scalars of the
proof become Python objects.

``Prover(setup, program)`` accepts the reference's ``Program`` (duck-typed: ``group_order``,
``common_preprocessed_input()``, ``wires()``, ``get_public_assignments()``).  For circuits that never
existed as ``Program`` objects (synthetic 2^k-gate circuits) use ``Prover.from_arrays`` and
``prove_arrays`` with numpy buffers."""
from __future__ import annotations

import ctypes
from dataclasses import dataclass, fields, make_dataclass
from typing import NamedTuple

import numpy as np

from . import _lib
from .curve import Scalar
from .custom_gates import is_next_row, padded, split_terms
from .lookup import check_lookup, check_lookups, padded_table, to_le_rows
from .field import CURVE_ORDER, FIELD_MODULUS, FQ
from .poly import Basis, _log2_exact, scalars_to_bytes
from .shuffle import check_shuffle
from .witness import WitnessReport
from .transcript import (KIND, LOOKUP, NEXT_ROW, SHUFFLE, Message1, Message2, Message3, Message4, Message5,
                         NextRowMessage4, NextRowShuffleMessage4, ShuffleMessage2, ShuffleMessage4, Transcript, blocks,
                         proof_bytes, proof_fields, schedule)

PK_ORDER = ("QM", "QL", "QR", "QO", "QC", "S1", "S2", "S3")  # compiler/program.py:10-30
PROOF_FIELDS = proof_fields()


def _encode(values) -> bytes:
    """a sequence of proof fields -> G1 points as x||y, every integer 32-byte big-endian"""
    out = bytearray()
    for v in values:
        if isinstance(v, tuple):
            out += v[0].n.to_bytes(32, "big") + v[1].n.to_bytes(32, "big")
        else:
            out += v.n.to_bytes(32, "big")
    return bytes(out)


def _decode(raw: bytes, names) -> dict:
    """32-byte big-endian words -> the fields ``names`` of the table (a point from two words, a scalar from one); a
    coordinate must be below q and a scalar below r, else ValueError naming the word by its index in the proof"""
    out, k = {}, 0
    for name in names:
        point = KIND[name] == "point"
        words = [int.from_bytes(raw[32 * w:32 * w + 32], "big") for w in range(k, k + (2 if point else 1))]
        for w, x in enumerate(words):
            if x >= (FIELD_MODULUS if point else CURVE_ORDER):
                raise ValueError("non-canonical proof encoding (word %d is not reduced)" % (k + w))
        out[name] = (FQ(words[0]), FQ(words[1])) if point else Scalar(words[0])
        k += len(words)
    return out


@dataclass
class Proof:
    msg_1: Message1
    msg_2: Message2
    msg_3: Message3
    msg_4: Message4
    msg_5: Message5

    BLOCKS, FIELDS, BYTES = (), (), proof_bytes()  # no fields beyond the plain 15

    def flatten(self):
        """prover.py:18-35."""
        out = {}
        for m in (self.msg_1, self.msg_2, self.msg_3, self.msg_4, self.msg_5):
            out.update((f.name, getattr(m, f.name)) for f in fields(m))
        return out

    def to_bytes(self) -> bytes:
        """Canonical 768-byte form: flatten() order, G1 as x||y, 32-byte big-endian integers."""
        return _encode(self.flatten().values())

    @classmethod
    def _from_values(cls, values: dict) -> "Proof":
        """the proof of the field values ``values`` (label -> value)"""
        return cls(*[m(*[values[f.name] for f in fields(m)]) for m in (Message1, Message2, Message3, Message4, Message5)])

    @classmethod
    def from_bytes(cls, raw: bytes) -> "Proof":
        """Inverse of to_bytes.  The encoding is canonical: coordinates must be below q and evaluations below r
        (ValueError otherwise) -- a second byte string for the same proof would make proofs malleable."""
        assert len(raw) == cls.BYTES
        return cls._from_values(_decode(raw, PROOF_FIELDS))


class _Extended:
    """A proof with extension blocks: ``plain`` (a ``Proof``), then the blocks' fields (``FIELDS``) in byte order.
    Encoded as the plain proof: flatten() order, G1 as x||y, 32-byte big-endian integers."""

    def flatten(self):
        out = self.plain.flatten()
        out.update((k, getattr(self, k)) for k in self.FIELDS)
        return out

    def to_bytes(self) -> bytes:
        return _encode(self.flatten().values())

    @classmethod
    def _from_values(cls, values: dict):
        return cls(Proof._from_values(values), *[values[k] for k in cls.FIELDS])

    @classmethod
    def from_bytes(cls, raw: bytes):
        """Inverse of to_bytes; ValueError for a word that is not reduced (coordinates below q, scalars below r)."""
        if len(raw) != cls.BYTES:
            raise ValueError("a %s proof has %d bytes, got %d" % (cls.NAME, cls.BYTES, len(raw)))
        return cls._from_values(_decode(raw, PROOF_FIELDS + cls.FIELDS))


def _proof_class(name: str, doc: str, **kind):
    """the proof class of a kind (``next_row``, ``shuffle``, ``lookup``): ``plain``, then its fields from the table"""
    ext = proof_fields(**kind)[len(PROOF_FIELDS):]
    return make_dataclass(name, [("plain", Proof)] + [(k, object) for k in ext], bases=(_Extended,), namespace={
        "__doc__": doc, "BLOCKS": blocks(**kind), "FIELDS": ext, "BYTES": proof_bytes(**kind),
        "NAME": " ".join(b.replace("_", "-") for b in blocks(**kind))})


LookupProof = _proof_class("LookupProof", """A proof with a lookup argument (plonkathon_b200/lookup.py): the plain proof's
    15 fields, then f_1 h1_1 h2_1 z2_1 and the six lookup evaluations (1216 bytes).""", lookup=True)
NextRowProof = _proof_class("NextRowProof", """A proof of a circuit with next-row custom gate terms
    (plonkathon_b200/custom_gates.py): the plain proof's 15 fields, then the wires at zeta w (864 bytes).""",
                            next_row=True)
ShuffleProof = _proof_class("ShuffleProof", """A proof of a circuit with a shuffle (plonkathon_b200/shuffle.py): the plain
    proof's 15 fields, then z3_1, qin_eval and z3_shifted_eval (896 bytes).""", shuffle=True)
NextRowShuffleProof = _proof_class("NextRowShuffleProof", """A proof of a circuit with a shuffle and next-row custom gate
    terms: the plain proof's 15 fields, the wires at zeta w, then the shuffle's three fields (992 bytes).""",
                                   next_row=True, shuffle=True)
LOOKUP_FIELDS, NEXT_ROW_FIELDS, SHUFFLE_FIELDS = LookupProof.FIELDS, NextRowProof.FIELDS, ShuffleProof.FIELDS
NEXT_ROW_PROOF_BYTES = NextRowProof.BYTES


class Kind(NamedTuple):
    """How a prover of one proof kind talks to the library (the layout itself is the table in transcript.py)."""
    proof: type       # its proof class
    suffix: str       # its entry points: pb200_prover_prove<suffix>, pb200_prover_round4<suffix>, ...
    round2: tuple     # (round-2 entry point, its message, the challenges it takes after beta and gamma)
    round4: tuple     # (round-4 entry point, its message)
    zk: str           # the zero-knowledge entry point
    blinders: int     # ... and its number of blinders

    @property
    def schedule(self) -> dict:
        return schedule(**{b: True for b in self.proof.BLOCKS})

    @property
    def device(self) -> str:
        """its whole-proof entry point for wire values already in device memory"""
        return "pb200_prover_prove_device" + self.suffix


_R2, _R4 = ("pb200_prover_round2", Message2, ()), ("pb200_prover_round4", Message4)
_R2_SHUFFLE = ("pb200_prover_round2_shuffle", ShuffleMessage2, ("theta", "kappa"))
# A lookup prover proves through prove_arrays only: its round-by-round path are the plain entry points, which the
# library refuses on it.
KINDS = {
    (): Kind(Proof, "", _R2, _R4, "pb200_prover_set_zk", 11),
    (NEXT_ROW,): Kind(NextRowProof, "_next_row", _R2, ("pb200_prover_round4_next_row", NextRowMessage4),
                      "pb200_prover_set_zk", 14),
    (SHUFFLE,): Kind(ShuffleProof, "_shuffle", _R2_SHUFFLE, ("pb200_prover_round4_shuffle", ShuffleMessage4),
                     "pb200_prover_set_zk_shuffle", 14),
    (NEXT_ROW, SHUFFLE): Kind(NextRowShuffleProof, "_next_row_shuffle", _R2_SHUFFLE,
                              ("pb200_prover_round4_next_row_shuffle", NextRowShuffleMessage4),
                              "pb200_prover_set_zk_shuffle", 17),
    (LOOKUP,): Kind(LookupProof, "_lookup", _R2, _R4, "pb200_prover_set_zk_lookup", 21),
}


def proof_kind(next_row=False, shuffle=False, lookup=False):
    """the kind of a prover or key with these blocks, or None for a combination without one"""
    return KINDS.get(blocks(next_row, shuffle, lookup))


def _as_le_rows(values, n) -> np.ndarray:
    """list of ints / Scalars, or an (m,32) uint8 / (m,8) uint32 array -> contiguous (n,32) uint8, zero padded."""
    if isinstance(values, np.ndarray):
        arr = np.ascontiguousarray(values).view(np.uint8).reshape(-1, 32)
    else:
        raw = b"".join((v.n if hasattr(v, "n") else int(v) % CURVE_ORDER).to_bytes(32, "little") for v in values)
        arr = np.frombuffer(raw, dtype=np.uint8).reshape(-1, 32)
    if arr.shape[0] < n:
        arr = np.concatenate([arr, np.zeros((n - arr.shape[0], 32), dtype=np.uint8)])
    assert arr.shape[0] == n
    return np.ascontiguousarray(arr)


def _is_cuda_tensor(x) -> bool:
    return type(x).__module__.startswith("torch") and getattr(x, "is_cuda", False)


def _wire_rows(name, values, n) -> np.ndarray:
    """a wire column as check_arrays takes it -> contiguous (n,32) uint8, zero padded; ValueError when malformed"""
    if isinstance(values, np.ndarray):
        if not ((values.dtype == np.uint8 and values.ndim == 2 and values.shape[1] == 32)
                or (values.dtype == np.uint32 and values.ndim == 2 and values.shape[1] == 8)):
            raise ValueError("%s must be an (m,32) uint8 or (m,8) uint32 array, got %s %s"
                             % (name, values.dtype, values.shape))
        m = values.shape[0]
    else:
        try:
            m = len(values)
        except TypeError:
            raise ValueError("%s must be a sequence of field elements or an array" % name) from None
    if m > n:
        raise ValueError("%s has %d rows, the circuit %d" % (name, m, n))
    return _as_le_rows(values, n)


def _pts(raw: bytes, count: int):
    return [(FQ(int.from_bytes(raw[64 * k:64 * k + 32], "little")),
             FQ(int.from_bytes(raw[64 * k + 32:64 * k + 64], "little"))) for k in range(count)]


def _raise(err: _lib.PlonkB200Error):
    if str(err).startswith("AssertionError"):
        raise AssertionError(str(err)) from None
    raise err


class Prover:
    _CREATE = "pb200_prover_create"
    _CREATE_CUSTOM = "pb200_prover_create_custom"
    _CREATE_NEXT_ROW = "pb200_prover_create_custom_next_row"
    next_row, _kind = False, KINDS[()]  # a plain prover until _create or a _set_* call says otherwise
    sharded = False  # one proof across several GPUs (parallel.ShardedProver)

    def __init__(self, setup, program):
        """prover.py:45-49."""
        self.group_order = program.group_order
        self.setup = setup
        self.program = program
        self.pk = program.common_preprocessed_input()
        cols = {k: scalars_to_bytes(getattr(self.pk, k).values) for k in PK_ORDER}
        self._create(setup, self.group_order, cols)

    @classmethod
    def from_arrays(cls, setup, group_order: int, pk_arrays: dict, ctx=None, custom=(), lookup=None, lookups=None,
                    shuffle=None):
        """pk_arrays: QM QL QR QO QC S1 S2 S3 -> list of ints or (n,32) uint8 little-endian arrays.
        ``ctx``: run this prover on another context (stream + scratch) of the same device than the setup's; the SRS
        is shared read-only, so several provers can be driven concurrently from different host threads.
        ``custom``: up to 4 custom gate terms ``((i, j, l), column)``, each adding ``Q_k a^i b^j c^l`` to the gate
        constraint (plonkathon_b200/custom_gates.py); ValueError for a malformed term.
        ``lookup``: ``(q_K, (t1, t2, t3))``, a lookup argument over one table of three columns
        (plonkathon_b200/lookup.py); ``prove_arrays`` then returns a 1216-byte ``LookupProof``.  ValueError for a
        malformed argument; the library refuses it on the sharded prover.
        ``lookups``: ``[(q_0, (t1, t2, t3)), (q_1, ...), ...]``, lookups over several tables told apart by a table tag
        (table k has id k; ``check_lookups``).  The proof is a ``LookupProof`` too.  Not together with ``lookup``.
        A custom term with six exponents ``((i, j, l, i', j', l'), column)`` may read the next row's wires; with one
        such term ``prove_arrays`` returns an 864-byte ``NextRowProof``.  Next-row terms do not combine with lookups
        (ValueError).
        ``shuffle``: ``(q_in, q_out)``, two boolean selectors with as many ones each: the rows with q_in = 1 hold the
        same multiset of (a, b, c) as the rows with q_out = 1 (plonkathon_b200/shuffle.py).  ``prove_arrays`` then returns
        an 896-byte ``ShuffleProof``, or a 992-byte ``NextRowShuffleProof`` with next-row terms.  ValueError for
        malformed selectors and for a shuffle with lookups.  Zero knowledge goes through ``set_zk_shuffle`` after the
        prover is made; ``set_zk`` refuses a shuffle prover."""
        if lookup is not None and lookups is not None:
            raise ValueError("pass either lookup= (one table) or lookups= (several tables), not both")
        if shuffle is not None and (lookup is not None or lookups is not None):
            raise ValueError("shuffles do not combine with lookups")
        custom = list(custom)
        if (lookup is not None or lookups is not None) and any(is_next_row(e) for e, _ in custom):
            raise ValueError("lookups do not combine with next-row custom gate terms")
        # before any device work
        lk = check_lookup(lookup, group_order) if lookup is not None else None
        lks = check_lookups(lookups, group_order) if lookups is not None else None
        sh = check_shuffle(shuffle, group_order) if shuffle is not None else None
        self = cls.__new__(cls)
        self.group_order = group_order
        self.setup = setup
        self.program = None
        self.pk = None
        cols = {k: _as_le_rows(pk_arrays[k], group_order) for k in PK_ORDER}
        self._create(setup, group_order, cols, ctx, custom)
        if lk is not None:
            self._set_lookup(*lk)
        if lks is not None:
            self._set_lookup_tagged(*lks)
        if sh is not None:
            self._set_shuffle(*sh)
        return self

    def _set_shuffle(self, q_in, q_out):
        keep = [to_le_rows(q_in), to_le_rows(q_out)]
        _lib.check(_lib.lib().pb200_prover_set_shuffle(self._h, *[k.ctypes.data_as(ctypes.c_void_p) for k in keep]))
        self._kind = proof_kind(next_row=self.next_row, shuffle=True)
        self._shuffle = tuple(k[:, 0] != 0 for k in keep)  # for WitnessReport's counts of a tuple on each side

    def _set_lookup(self, qk, cols, rows):
        keep = [to_le_rows(qk)] + [to_le_rows(c) for c in cols]
        ptr = [k.ctypes.data_as(ctypes.c_void_p) for k in keep]
        _lib.check(_lib.lib().pb200_prover_set_lookup(self._h, *ptr, rows))
        self._kind = proof_kind(lookup=True)

    def _set_lookup_tagged(self, qk, qtag, cols, rows):
        """cols: t1, t2, t3, t4 (the table ids)"""
        keep = [to_le_rows(qk), to_le_rows(qtag)] + [to_le_rows(c) for c in cols]
        ptr = [k.ctypes.data_as(ctypes.c_void_p) for k in keep]
        _lib.check(_lib.lib().pb200_prover_set_lookup_tagged(self._h, *ptr, rows))
        self._kind = proof_kind(lookup=True)

    def _create(self, setup, n, cols, ctx=None, custom=()):
        exps, ccols = split_terms(custom, n)  # before any device work: a malformed term is a ValueError
        self.ctx = ctx or setup.ctx
        self._log_n = _log2_exact(n)
        self.custom_exponents = exps
        self.next_row = any(is_next_row(e) for e in exps)
        self._kind = proof_kind(next_row=self.next_row)
        keep = [c if isinstance(c, bytes) else c.tobytes() for c in (cols[k] for k in PK_ORDER)]
        arr = (ctypes.c_char_p * 8)(*keep)
        h = ctypes.c_void_p()
        if exps:
            ckeep = [_as_le_rows(col, n).tobytes() for col in ccols]
            carr = (ctypes.c_char_p * len(ckeep))(*ckeep)
            if self.next_row:  # six bytes per term
                ebytes = bytes(x for e in exps for x in padded(e))
                create = getattr(_lib.lib(), self._CREATE_NEXT_ROW)
            else:  # three bytes per term: the same-row path
                ebytes = bytes(x for e in exps for x in padded(e)[:3])
                create = getattr(_lib.lib(), self._CREATE_CUSTOM)
            _lib.check(create(self.ctx.handle, setup._srs, self._log_n, ctypes.cast(arr, ctypes.c_void_p), len(exps),
                              ebytes, ctypes.cast(carr, ctypes.c_void_p), ctypes.byref(h)))
        else:
            create = getattr(_lib.lib(), self._CREATE)  # the multi-GPU prover creates its sharded counterpart
            _lib.check(create(self.ctx.handle, setup._srs, self._log_n, ctypes.cast(arr, ctypes.c_void_p),
                              ctypes.byref(h)))
        self._h = h

    @property
    def sliced(self) -> bool:
        """True when the library chose (or ``PB200_SLICED=1`` forced) the sliced round 3: the cache on the 4n coset did
        not fit the free device memory, so the quotient is evaluated one n-point slice of the coset at a time.  Same
        proofs; zero knowledge, lookups, shuffles and next-row terms are refused on such a prover."""
        out = ctypes.c_int()
        _lib.check(_lib.lib().pb200_prover_sliced(self._h, ctypes.byref(out)))
        return bool(out.value)

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().pb200_prover_destroy(self._h)
                self._h = None
        except Exception:
            pass

    def _call(self, entry: str, *args):
        """one C-ABI call on this prover; a failed assertion of the witness becomes an AssertionError"""
        try:
            _lib.check(getattr(_lib.lib(), entry)(self._h, *args))
        except _lib.PlonkB200Error as e:
            _raise(e)

    # ------------------------------------------------------------------ array-level fast path
    def prove_arrays(self, A, B, C, public) -> bytes:
        """One C-ABI call for the whole proof (rounds 1-5 + transcript); returns the canonical bytes of the prover's
        proof kind: 768 for a ``Proof``, 1216 for a ``LookupProof`` (lookup argument), 864 for a ``NextRowProof``
        (next-row custom gate terms), 896 (992) for a ``ShuffleProof`` (``NextRowShuffleProof``).
        A, B, C may also be contiguous (n, 32) uint8 CUDA tensors on the prover's device (``solve_wires(device=True)``),
        which are read where they are; ValueError for malformed tensors and on the sharded prover."""
        n = self.group_order
        pub = _as_le_rows(public, len(public)) if len(public) else np.zeros((0, 32), dtype=np.uint8)
        out = ctypes.create_string_buffer(self._kind.proof.BYTES)
        ptrs = self._device_wires(A, B, C)
        if ptrs is not None:
            if self.sharded:
                raise ValueError("the sharded prover takes wire values in host memory, not CUDA tensors")
            self._call(self._kind.device, *ptrs, pub.ctypes.data_as(ctypes.c_void_p), pub.shape[0], out)
            return out.raw
        a, b, c = (_as_le_rows(v, n) for v in (A, B, C))
        self._call("pb200_prover_prove" + self._kind.suffix, *[x.ctypes.data_as(ctypes.c_void_p) for x in (a, b, c, pub)],
                   pub.shape[0], out)
        return out.raw

    def _device_wires(self, A, B, C):
        """pointers to A, B, C when they are CUDA tensors, checked and with their stream synchronised (the library
        runs on its own stream); None for host values; ValueError for a mix or a malformed tensor"""
        n = self.group_order
        on_device = [_is_cuda_tensor(X) for X in (A, B, C)]
        if any(on_device) and not all(on_device):
            raise ValueError("A, B and C must all be CUDA tensors or all be host values")
        if not all(on_device):
            return None
        for name, X in zip("ABC", (A, B, C)):
            if tuple(X.shape) != (n, 32) or str(X.dtype) != "torch.uint8" or not X.is_contiguous():
                raise ValueError("%s must be a contiguous (%d, 32) uint8 tensor, got %s %s"
                                 % (name, n, tuple(X.shape), X.dtype))
            if X.device.index != self.ctx.device:
                raise ValueError("%s is on cuda:%s, the prover on cuda:%d" % (name, X.device.index, self.ctx.device))
        import torch
        for X in (A, B, C):
            torch.cuda.current_stream(X.device).synchronize()
        return [ctypes.c_void_p(X.data_ptr()) for X in (A, B, C)]

    # ------------------------------------------------------------------ witness check
    def check_arrays(self, A, B, C, public, limit: int = 16) -> WitnessReport:
        """Check a witness against this prover's key without proving: every failing gate, copy constraint, lookup row
        and shuffle row, each category as an exact count and its lowest ``limit`` locations (``WitnessReport``).  The
        report is empty iff rounds 1 and 2 of ``prove_arrays`` pass their checks.  Draws no blinders and changes no
        later proof.  A, B, C as for ``prove_arrays`` (lists of ints, or (m,32) uint8 / (m,8) uint32 arrays, m <= n,
        zero padded), or (n,32) uint8 CUDA tensors on the prover's device, which stay there.  The first check of a
        prover builds the copy permutation on the device and keeps it (12 bytes a row).  ValueError for malformed
        inputs, before the library is called; the library refuses values not reduced below r and the sharded
        prover."""
        return self._check(A, B, C, public, limit)

    def _check(self, A, B, C, public, limit, names=None) -> WitnessReport:
        """check_arrays; names(row, col) -> the variable of a cell, for this report only"""
        n = self.group_order
        if isinstance(limit, bool) or not isinstance(limit, (int, np.integer)) or not 0 <= limit <= 3 * n:
            raise ValueError("limit must be an integer in [0, 3n = %d], got %r" % (3 * n, limit))
        limit = int(limit)
        if len(public) > n:
            raise ValueError("%d public inputs for %d rows" % (len(public), n))
        ptrs = self._device_wires(A, B, C)
        if ptrs is not None:
            entry, wires = "pb200_prover_check_device", None
        else:
            wires = tuple(_wire_rows(name, X, n) for name, X in zip("ABC", (A, B, C)))
            ptrs = [w.ctypes.data_as(ctypes.c_void_p) for w in wires]
            entry = "pb200_prover_check"
        pub = _as_le_rows([int(x) % CURVE_ORDER for x in public], len(public)) if len(public) else \
            np.zeros((0, 32), np.uint8)
        counts = (ctypes.c_uint64 * 5)()
        lists = (ctypes.c_uint32 * max(1, 6 * limit))()
        _lib.check(getattr(_lib.lib(), entry)(self._h, *ptrs, pub.ctypes.data_as(ctypes.c_void_p), pub.shape[0], limit,
                                               counts, lists))
        if wires is None and any(counts):  # the values the report prints
            wires = tuple(X.cpu().numpy() for X in (A, B, C))
        return WitnessReport._from_library(counts, lists[:6 * limit], limit, wires, getattr(self, "_shuffle", None),
                                           names)

    def check(self, witness, limit: int = 16) -> WitnessReport:
        """``check_arrays`` for a prover made from a reference ``Program``, with the witness dict ``prove`` takes; the
        report names each copy-constraint cell by its variable (``program.wires()``)."""
        if self.program is None:
            raise ValueError("check(witness) needs a prover made from a Program; use check_arrays")
        A, B, C, public = self._witness_columns(witness)
        wires = self.program.wires()
        return self._check(A, B, C, public, limit,
                           lambda row, col: getattr(wires[row], "LRO"[col]) if row < len(wires) else None)

    # ------------------------------------------------------------------ the reference's surface
    def prove(self, witness) -> Proof:
        """prover.py:51-84, following the schedule of the prover's kind (transcript.py) and returning its proof class:
        a ``NextRowProof`` with next-row custom gate terms, a ``ShuffleProof`` (``NextRowShuffleProof``) with a
        shuffle."""
        kind = self._kind
        transcript = Transcript(b"plonk")
        msg_1 = self.round_1(witness)  # also collects the public inputs (prover.py:57-62)
        for name, value in zip(kind.schedule["1"][2], transcript.round_1(msg_1, kind.schedule)):
            setattr(self, name, value)  # beta, gamma (and theta, kappa with a shuffle)
        msg_2 = self.round_2()
        self.alpha, self.fft_cofactor = transcript.round_2(msg_2)
        msg_3 = self.round_3()
        self.zeta = transcript.round_3(msg_3)
        msg_4 = self.round_4()
        self.v = transcript.round_4(msg_4)
        msg_5 = self.round_5()
        values = {}
        for m in (msg_1, msg_2, msg_3, msg_4, msg_5):
            values.update((f.name, getattr(m, f.name)) for f in fields(m))
        return kind.proof._from_values(values)

    def _witness_columns(self, witness):
        """prover.py:86-103: a witness dict (variable -> value) -> the wire columns A, B, C and the public inputs"""
        if None not in witness:
            witness[None] = 0
        wires = self.program.wires()
        A = [int(witness[w.L]) % CURVE_ORDER for w in wires]
        B = [int(witness[w.R]) % CURVE_ORDER for w in wires]
        C = [int(witness[w.O]) % CURVE_ORDER for w in wires]
        return A, B, C, [int(witness[v]) % CURVE_ORDER for v in self.program.get_public_assignments()]

    def round_1(self, witness) -> Message1:
        """prover.py:86-119."""
        A, B, C, self._public = self._witness_columns(witness)
        return self.round_1_arrays(A, B, C, self._public)

    def round_1_arrays(self, A, B, C, public) -> Message1:
        """round 1 from wire-value columns (lists of ints or (n,32) uint8 arrays) instead of a witness dict"""
        n = self.group_order
        self._public = [int(x) % CURVE_ORDER for x in public]
        a, b, c = (_as_le_rows(v, n) for v in (A, B, C))
        pub = _as_le_rows(self._public, len(self._public)) if self._public else np.zeros((0, 32), np.uint8)
        out = ctypes.create_string_buffer(192)
        self._call("pb200_prover_round1", *[x.ctypes.data_as(ctypes.c_void_p) for x in (a, b, c, pub)], pub.shape[0], out)
        return Message1(*self._commitments(0, 3, out.raw))

    @staticmethod
    def _le(x) -> bytes:
        return (int(x) % CURVE_ORDER).to_bytes(32, "little")

    def round_2(self) -> Message2:
        """prover.py:121-152.  A shuffle prover returns a ``ShuffleMessage2`` (z_1, z3_1) and needs ``theta`` and
        ``kappa`` set beside ``beta`` and ``gamma``."""
        entry, message, extra = self._kind.round2
        out = ctypes.create_string_buffer(64 * len(fields(message)))
        self._call(entry, *[self._le(getattr(self, c)) for c in ("beta", "gamma") + extra], out)
        return message(*self._commitments(3, len(fields(message)), out.raw))

    def round_3(self) -> Message3:
        """prover.py:154-226."""
        out = ctypes.create_string_buffer(192)
        self._call("pb200_prover_round3", self._le(self.alpha), self._le(self.fft_cofactor), out)
        return Message3(*self._commitments(4, 3, out.raw))

    def round_4(self) -> Message4:
        """prover.py:228-239.  A next-row prover returns a ``NextRowMessage4``: the six evaluations, then a, b, c at
        zeta w (NEXT_ROW_SCHEDULE).  A shuffle prover returns a ``ShuffleMessage4`` or ``NextRowShuffleMessage4``, with
        q_in(zeta) and Z3(zeta w) last."""
        entry, message = self._kind.round4
        count = len(fields(message))
        out = ctypes.create_string_buffer(32 * count)
        self._call(entry, self._le(self.zeta), out)
        return message(*[Scalar(int.from_bytes(out.raw[32 * k:32 * k + 32], "little")) for k in range(count)])

    def round_5(self) -> Message5:
        """prover.py:241-306."""
        out = ctypes.create_string_buffer(128)
        self._call("pb200_prover_round5", self._le(self.v), out)
        return Message5(*self._commitments(7, 2, out.raw))

    # ------------------------------------------------------------------ round state (prover.py: self.A .. self.T3)
    def _state(self, which: int, basis):
        """a vector of the device-resident round state as a lazily materialised Polynomial (stays in HBM)"""
        import torch
        from .poly import Polynomial
        n = self.group_order
        t = torch.empty((n, 32), dtype=torch.uint8, device=torch.device("cuda", self.ctx.device))
        _lib.check(_lib.lib().pb200_prover_read_vector(self._h, which, ctypes.c_void_p(t.data_ptr())))
        return Polynomial(None, basis, _dev=t)

    A = property(lambda self: self._state(0, Basis.LAGRANGE), doc="prover.py:97-103 (after round_1)")
    B = property(lambda self: self._state(1, Basis.LAGRANGE))
    C = property(lambda self: self._state(2, Basis.LAGRANGE))
    Z = property(lambda self: self._state(3, Basis.LAGRANGE), doc="prover.py:147 (after round_2)")
    PI = property(lambda self: self._state(4, Basis.LAGRANGE), doc="prover.py:57-63 (after round_1)")
    # T1, T2, T3 are Lagrange-basis Polynomials in the reference (prover.py:209-219): the forward transform of the
    # three coefficient thirds the library keeps (after round_3)
    def _piece(self, which: int, name: str):
        if getattr(self, "zk", False):
            raise RuntimeError("%s is not available in zero-knowledge mode: the blinded quotient pieces have n + 1, "
                               "n + 1 and n + 6 (or n + 9) coefficients, so they have no n-value Lagrange form" % name)
        return self._state(which, Basis.MONOMIAL).fft(ctx=self.ctx)

    T1 = property(lambda self: self._piece(5, "T1"))
    T2 = property(lambda self: self._piece(6, "T2"))
    T3 = property(lambda self: self._piece(7, "T3"))

    # ------------------------------------------------------------------ zero knowledge
    def _set_zk(self, block, what: str, enable: bool, blinders):
        """the body of set_zk (block None), set_zk_lookup and set_zk_shuffle: the blinders of the kind that entry point
        serves, checked here, then the library's own checks"""
        kind = proof_kind(next_row=self.next_row and block != LOOKUP, shuffle=block == SHUFFLE, lookup=block == LOOKUP)
        raw = None
        if enable and blinders is not None:
            blinders = [int(b) for b in blinders]
            if len(blinders) != kind.blinders:
                raise ValueError("%s %d blinders b1..b%d%s, got %d" % (
                    what, kind.blinders, kind.blinders,
                    " on a prover with next-row terms" if NEXT_ROW in kind.proof.BLOCKS else "", len(blinders)))
            if any(not 0 <= b < CURVE_ORDER for b in blinders):
                raise ValueError("zero-knowledge blinders must lie in [0, r)")
            raw = b"".join(b.to_bytes(32, "little") for b in blinders)
        _lib.check(getattr(_lib.lib(), kind.zk)(self._h, 1 if enable else 0, raw))
        self.zk = bool(enable)

    def set_zk(self, enable: bool = True, blinders=None):
        """Zero-knowledge mode for every later proof: A, B, C, Z and the quotient pieces are blinded as in the PLONK
        paper (eprint 2019/953), with 11 scalars b1..b11 per proof.  The proof keeps its 768 bytes and the verifier does
        not change.  ``blinders=None``: fresh scalars from the OS CSPRNG for every proof; otherwise 11 integers in
        [0, r) used for every proof (reproducible tests only: fixed blinders reveal the witness to whoever knows them).
        Needs n >= 8 and an SRS of at least n + 6 powers; the sharded prover has no zero-knowledge mode.
        A prover with next-row custom gate terms takes 14 blinders: b12, b13, b14 give A, B, C a third one, since they
        are opened at zeta and at zeta w (DESIGN.md section 1).  It needs n >= 16 and an SRS of n + 9 powers."""
        self._set_zk(None, "zero knowledge takes", enable, blinders)

    def set_zk_lookup(self, enable: bool = True, blinders=None):
        """Zero-knowledge mode for the later proofs of a lookup prover (``lookup=`` or ``lookups=``): ``set_zk``'s
        blinding and 10 more scalars for F, H1, H2 and Z2, 21 in all (DESIGN.md section 1).  The proofs keep their 1216
        bytes and the verifier does not change.  ``blinders=None``: fresh scalars from the OS CSPRNG for every proof;
        otherwise 21 integers in [0, r) used for every proof (reproducible tests only).  ``enable=False`` (or
        ``set_zk(False)``) returns to plain lookup proofs.  Needs a lookup table, n >= 8 and an SRS of n + 6 powers."""
        self._set_zk(LOOKUP, "zero-knowledge lookups take", enable, blinders)

    def set_zk_shuffle(self, enable: bool = True, blinders=None):
        """Zero-knowledge mode for the later proofs of a shuffle prover (``shuffle=``): ``set_zk``'s blinding and 3 more
        scalars for Z3, the last three: 14 in all, 17 with next-row custom gate terms (DESIGN.md section 1).  The proofs
        keep their 896 (992) bytes and the verifier does not change.  ``blinders=None``: fresh scalars from the OS CSPRNG
        for every proof; otherwise 14 (17) integers in [0, r) used for every proof (reproducible tests only).
        ``enable=False`` (or ``set_zk(False)``) returns to plain shuffle proofs.  Needs a shuffle, n >= 8 and an SRS of
        n + 6 powers (n >= 16 and n + 9 powers with next-row terms)."""
        self._set_zk(SHUFFLE, "zero-knowledge shuffles take", enable, blinders)

    def _commitments(self, first_slot: int, count: int, raw: bytes):
        """commitments a round produced"""
        return _pts(raw, count)

    def fft_expand(self, x):
        """prover.py:308-309 -- x.to_coset_extended_lagrange(self.fft_cofactor)."""
        return x.to_coset_extended_lagrange(self.fft_cofactor, ctx=self.ctx)

    def expanded_evals_to_coeffs(self, x):
        """prover.py:311-312 -- x.coset_extended_lagrange_to_coeffs(self.fft_cofactor)."""
        return x.coset_extended_lagrange_to_coeffs(self.fft_cofactor, ctx=self.ctx)

    def rlc(self, term_1, term_2):
        """prover.py:314-315."""
        return term_1 + term_2 * self.beta + self.gamma
