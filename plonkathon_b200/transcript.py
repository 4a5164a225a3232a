"""Drop-in for the reference's ``transcript.py``: the five message records (transcript.py:8-55) and
``Transcript`` (transcript.py:58-123).  The Merlin/STROBE/Keccak machinery is host code inside
libplonk_b200.so (csrc/transcript.cuh); this module binds it and holds the proof layout as one table, from which
every proof kind's per-round schedule follows: which fields are absorbed (points as x then y, scalars, all 32-byte
big-endian) and which challenges are drawn afterwards."""
from __future__ import annotations

import ctypes
from dataclasses import make_dataclass

from . import _lib
from .curve import Scalar

# The proof layout: every field of every proof kind as (label, kind, step, block), in byte order -- the plain proof's 15
# fields in ``Proof.flatten()`` order, then the next-row block (plonkathon_b200/custom_gates.py), the shuffle block
# (plonkathon_b200/shuffle.py) and the lookup block (plonkathon_b200/lookup.py).  The label is the transcript label and
# the proof classes' attribute; a point is 64 bytes (x then y), a scalar 32.  A prover or key has a set of blocks, and
# its proof is this table filtered to the plain block and those blocks.  One table gives both orders because
#
#     within each transcript step, the fields are absorbed in byte order.
#
# csrc/proof_layout.cuh holds the same table for the library (tests/test_proof_layout.py compares the two).
PLAIN, NEXT_ROW, SHUFFLE, LOOKUP = "plain", "next_row", "shuffle", "lookup"
STEPS = ("1", "1L", "2", "3", "4", "5")  # 1L: the lookup commitments, between rounds 1 and 2
FIELDS = (
    ("a_1", "point", "1", PLAIN), ("b_1", "point", "1", PLAIN), ("c_1", "point", "1", PLAIN),
    ("z_1", "point", "2", PLAIN),
    ("t_lo_1", "point", "3", PLAIN), ("t_mid_1", "point", "3", PLAIN), ("t_hi_1", "point", "3", PLAIN),
    ("a_eval", "scalar", "4", PLAIN), ("b_eval", "scalar", "4", PLAIN), ("c_eval", "scalar", "4", PLAIN),
    ("s1_eval", "scalar", "4", PLAIN), ("s2_eval", "scalar", "4", PLAIN), ("z_shifted_eval", "scalar", "4", PLAIN),
    ("W_z_1", "point", "5", PLAIN), ("W_zw_1", "point", "5", PLAIN),
    ("a_shifted_eval", "scalar", "4", NEXT_ROW), ("b_shifted_eval", "scalar", "4", NEXT_ROW),
    ("c_shifted_eval", "scalar", "4", NEXT_ROW),
    ("z3_1", "point", "2", SHUFFLE), ("qin_eval", "scalar", "4", SHUFFLE), ("z3_shifted_eval", "scalar", "4", SHUFFLE),
    ("f_1", "point", "1L", LOOKUP), ("h1_1", "point", "1L", LOOKUP), ("h2_1", "point", "1L", LOOKUP),
    ("z2_1", "point", "2", LOOKUP),
    ("f_eval", "scalar", "4", LOOKUP), ("t_eval", "scalar", "4", LOOKUP), ("t_shifted_eval", "scalar", "4", LOOKUP),
    ("h2_eval", "scalar", "4", LOOKUP), ("h1_shifted_eval", "scalar", "4", LOOKUP),
    ("z2_shifted_eval", "scalar", "4", LOOKUP),
)
KIND = {label: kind for label, kind, _, _ in FIELDS}
# the challenges each step draws after absorbing its fields, in drawing order, as (label, step, block)
CHALLENGES = (
    ("beta", "1", PLAIN), ("gamma", "1", PLAIN), ("theta", "1", SHUFFLE), ("kappa", "1", SHUFFLE), ("eta", "1", LOOKUP),
    ("delta", "1L", LOOKUP), ("epsilon", "1L", LOOKUP), ("alpha", "2", PLAIN), ("fft_cofactor", "2", PLAIN),
    ("zeta", "3", PLAIN), ("v", "4", PLAIN), ("u", "5", PLAIN),
)


def blocks(next_row=False, shuffle=False, lookup=False) -> tuple:
    """the extension blocks of a proof kind, in table order"""
    return tuple(b for b, on in ((NEXT_ROW, next_row), (SHUFFLE, shuffle), (LOOKUP, lookup)) if on)


def proof_fields(next_row=False, shuffle=False, lookup=False) -> tuple:
    """the labels of a kind's proof fields in byte order"""
    have = (PLAIN,) + blocks(next_row, shuffle, lookup)
    return tuple(label for label, _, _, block in FIELDS if block in have)


def proof_bytes(next_row=False, shuffle=False, lookup=False) -> int:
    return sum(64 if KIND[f] == "point" else 32 for f in proof_fields(next_row, shuffle, lookup))


def schedule(next_row=False, shuffle=False, lookup=False) -> dict:
    """step -> (the step's fields in absorption order, their kind, the challenges drawn afterwards) for one proof kind;
    a step with neither (1L without lookups) is left out"""
    have = (PLAIN,) + blocks(next_row, shuffle, lookup)
    out = {}
    for step in STEPS:
        fields = [(label, kind) for label, kind, s, block in FIELDS if s == step and block in have]
        drawn = tuple(label for label, s, block in CHALLENGES if s == step and block in have)
        if fields:
            kinds = {kind for _, kind in fields}
            assert len(kinds) == 1, "a step absorbs fields of one kind"
            out[step] = (tuple(label for label, _ in fields), kinds.pop(), drawn)
    return out


SCHEDULE = schedule()
LOOKUP_SCHEDULE = schedule(lookup=True)
NEXT_ROW_SCHEDULE = schedule(next_row=True)
SHUFFLE_SCHEDULE = schedule(shuffle=True)
NEXT_ROW_SHUFFLE_SCHEDULE = schedule(next_row=True, shuffle=True)

# message class -> the schedule it follows (Transcript.round_2, round_4; SCHEDULE for any other record)
_SCHEDULE_OF = {}


def _message(name: str, sched: dict, step: str):
    cls = make_dataclass(name, [(label, object) for label in sched[step][0]])
    _SCHEDULE_OF[cls] = sched
    return cls


# Message1 .. Message5: plain records with exactly the reference's field names and order
Message1, Message2, Message3, Message4, Message5 = (_message("Message" + s, SCHEDULE, s) for s in "12345")
# round 4 of a next-row prover: Message4's fields, then the three shifted wire evaluations
NextRowMessage4 = _message("NextRowMessage4", NEXT_ROW_SCHEDULE, "4")
# rounds 2 and 4 of a shuffle prover (round 4 with and without next-row terms)
ShuffleMessage2 = _message("ShuffleMessage2", SHUFFLE_SCHEDULE, "2")
ShuffleMessage4 = _message("ShuffleMessage4", SHUFFLE_SCHEDULE, "4")
NextRowShuffleMessage4 = _message("NextRowShuffleMessage4", NEXT_ROW_SHUFFLE_SCHEDULE, "4")


def _as_int(x) -> int:
    return x.n if hasattr(x, "n") else int(x)


class Transcript:
    def __init__(self, label: bytes):
        handle = ctypes.c_void_p()
        _lib.check(_lib.lib().pb200_transcript_create(label, len(label), ctypes.byref(handle)))
        self._h = handle

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                _lib.lib().pb200_transcript_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ---- the MerlinTranscript surface the reference's class inherits (transcript.py:3,58)
    def append_message(self, label: bytes, message: bytes) -> None:
        _lib.check(_lib.lib().pb200_transcript_append_message(self._h, label, len(label), message, len(message)))

    def challenge_bytes(self, label: bytes, length: int) -> bytes:
        buf = ctypes.create_string_buffer(length)
        _lib.check(_lib.lib().pb200_transcript_challenge_bytes(self._h, label, len(label), buf, length))
        return buf.raw

    # ---- transcript.py:59-75
    append = append_message

    def append_scalar(self, label: bytes, item) -> None:
        self.append_message(label, _as_int(item).to_bytes(32, "big"))

    def append_point(self, label: bytes, item) -> None:
        for coordinate in (item[0], item[1]):  # the identity (None) is unsupported, as in the reference
            self.append_message(label, _as_int(coordinate).to_bytes(32, "big"))

    def get_and_append_challenge(self, label: bytes) -> Scalar:
        """255 squeezed bytes as a big-endian integer mod r, redrawn while zero, then re-absorbed under the
        same label -- all inside the library."""
        out = ctypes.create_string_buffer(32)
        _lib.check(_lib.lib().pb200_transcript_get_and_append_challenge(self._h, label, len(label), out))
        return Scalar(int.from_bytes(out.raw, "little"))

    # ---- transcript.py:77-123
    def _round(self, step: str, message, schedule: dict = None):
        fields, kind, challenges = (schedule or _SCHEDULE_OF.get(type(message), SCHEDULE))[step]
        absorb = self.append_point if kind == "point" else self.append_scalar
        for name in fields:
            absorb(name.encode(), getattr(message, name))
        drawn = tuple(self.get_and_append_challenge(c.encode()) for c in challenges)
        return drawn if len(drawn) > 1 else drawn[0]

    def replay(self, schedule: dict, values: dict) -> dict:
        """every step of ``schedule`` in order over ``values`` (field name -> point or scalar); -> {label: challenge}"""
        drawn = {}
        for fields, kind, challenges in schedule.values():
            absorb = self.append_point if kind == "point" else self.append_scalar
            for name in fields:
                absorb(name.encode(), values[name])
            for c in challenges:
                drawn[c] = self.get_and_append_challenge(c.encode())
        return drawn

    def round_1(self, message, schedule: dict = SCHEDULE):
        """``schedule=SHUFFLE_SCHEDULE`` draws theta and kappa after beta and gamma (four challenges)"""
        return self._round("1", message, schedule)

    def round_2(self, message):
        """the schedule of the message's type: a ``ShuffleMessage2`` follows SHUFFLE_SCHEDULE"""
        return self._round("2", message)

    def round_3(self, message):
        return self._round("3", message)

    def round_4(self, message):
        """the schedule of the message's type: a ``NextRowMessage4`` follows NEXT_ROW_SCHEDULE, a ``ShuffleMessage4``
        SHUFFLE_SCHEDULE and a ``NextRowShuffleMessage4`` NEXT_ROW_SHUFFLE_SCHEDULE"""
        return self._round("4", message)

    def round_5(self, message):
        return self._round("5", message)
