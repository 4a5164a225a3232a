"""Drop-in for the reference's ``transcript.py``: the five message records (transcript.py:8-55) and
``Transcript`` (transcript.py:58-123).  The Merlin/STROBE/Keccak machinery is host code inside
libplonk_b200.so (csrc/transcript.cuh); this module binds it and lays the reference's per-round schedule out
as a table: which fields of a message are absorbed (points as x then y, scalars, all 32-byte big-endian) and
which challenges are drawn afterwards."""
from __future__ import annotations

import ctypes
from dataclasses import make_dataclass

from . import _lib
from .curve import Scalar

# round -> (message field names in absorption order, kind of those fields, challenge labels drawn afterwards)
SCHEDULE = {
    1: (("a_1", "b_1", "c_1"), "point", ("beta", "gamma")),
    2: (("z_1",), "point", ("alpha", "fft_cofactor")),
    3: (("t_lo_1", "t_mid_1", "t_hi_1"), "point", ("zeta",)),
    4: (("a_eval", "b_eval", "c_eval", "s1_eval", "s2_eval", "z_shifted_eval"), "scalar", ("v",)),
    5: (("W_z_1", "W_zw_1"), "point", ("u",)),
}

# The same table for a proof with a lookup argument (plonkathon_b200/lookup.py): step 1 also draws eta, step 1L absorbs
# the lookup commitments, round 2 absorbs Z2 beside Z and round 4 the six lookup evaluations after the plain ones.
LOOKUP_SCHEDULE = {
    "1": (("a_1", "b_1", "c_1"), "point", ("beta", "gamma", "eta")),
    "1L": (("f_1", "h1_1", "h2_1"), "point", ("delta", "epsilon")),
    "2": (("z_1", "z2_1"), "point", ("alpha", "fft_cofactor")),
    "3": (("t_lo_1", "t_mid_1", "t_hi_1"), "point", ("zeta",)),
    "4": (("a_eval", "b_eval", "c_eval", "s1_eval", "s2_eval", "z_shifted_eval", "f_eval", "t_eval", "t_shifted_eval",
           "h2_eval", "h1_shifted_eval", "z2_shifted_eval"), "scalar", ("v",)),
    "5": (("W_z_1", "W_zw_1"), "point", ("u",)),
}

# The same table for a proof with next-row custom gate terms (plonkathon_b200/custom_gates.py): round 4 also absorbs the
# wires at zeta w, after z_shifted_eval and before v is drawn.
NEXT_ROW_SCHEDULE = dict(SCHEDULE)
NEXT_ROW_SCHEDULE[4] = (SCHEDULE[4][0] + ("a_shifted_eval", "b_shifted_eval", "c_shifted_eval"), "scalar", ("v",))

# The same table for a proof with a shuffle (plonkathon_b200/shuffle.py): step 1 also draws theta and kappa (no commitment
# before them), step 2 absorbs Z3 beside Z and step 4 q_in(zeta) and Z3(zeta w) last.  NEXT_ROW_SHUFFLE_SCHEDULE is the
# form for a circuit with next-row custom gate terms: the three shifted wire evaluations come before the shuffle's two.
SHUFFLE_FIELDS_4 = ("qin_eval", "z3_shifted_eval")
SHUFFLE_SCHEDULE = dict(SCHEDULE)
SHUFFLE_SCHEDULE[1] = (SCHEDULE[1][0], "point", ("beta", "gamma", "theta", "kappa"))
SHUFFLE_SCHEDULE[2] = (("z_1", "z3_1"), "point", SCHEDULE[2][2])
SHUFFLE_SCHEDULE[4] = (SCHEDULE[4][0] + SHUFFLE_FIELDS_4, "scalar", ("v",))
NEXT_ROW_SHUFFLE_SCHEDULE = dict(SHUFFLE_SCHEDULE)
NEXT_ROW_SHUFFLE_SCHEDULE[4] = (NEXT_ROW_SCHEDULE[4][0] + SHUFFLE_FIELDS_4, "scalar", ("v",))

# Message1 .. Message5: plain records with exactly the reference's field names and order
Message1, Message2, Message3, Message4, Message5 = (
    make_dataclass("Message%d" % rnd, [(name, object) for name in SCHEDULE[rnd][0]]) for rnd in sorted(SCHEDULE))
# round 4 of a next-row prover: Message4's fields, then the three shifted wire evaluations
NextRowMessage4 = make_dataclass("NextRowMessage4", [(name, object) for name in NEXT_ROW_SCHEDULE[4][0]])
# rounds 2 and 4 of a shuffle prover (round 4 with and without next-row terms)
ShuffleMessage2 = make_dataclass("ShuffleMessage2", [(name, object) for name in SHUFFLE_SCHEDULE[2][0]])
ShuffleMessage4 = make_dataclass("ShuffleMessage4", [(name, object) for name in SHUFFLE_SCHEDULE[4][0]])
NextRowShuffleMessage4 = make_dataclass("NextRowShuffleMessage4",
                                        [(name, object) for name in NEXT_ROW_SHUFFLE_SCHEDULE[4][0]])


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
    def _round(self, rnd: int, message, schedule: dict = SCHEDULE):
        fields, kind, challenges = schedule[rnd]
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
        return self._round(1, message, schedule)

    def round_2(self, message):
        """a ``ShuffleMessage2`` follows SHUFFLE_SCHEDULE"""
        return self._round(2, message, SHUFFLE_SCHEDULE if isinstance(message, ShuffleMessage2) else SCHEDULE)

    def round_3(self, message):
        return self._round(3, message)

    def round_4(self, message):
        """a ``NextRowMessage4`` follows NEXT_ROW_SCHEDULE, a ``ShuffleMessage4`` SHUFFLE_SCHEDULE and a
        ``NextRowShuffleMessage4`` NEXT_ROW_SHUFFLE_SCHEDULE"""
        schedule = {NextRowMessage4: NEXT_ROW_SCHEDULE, ShuffleMessage4: SHUFFLE_SCHEDULE,
                    NextRowShuffleMessage4: NEXT_ROW_SHUFFLE_SCHEDULE}.get(type(message), SCHEDULE)
        return self._round(4, message, schedule)

    def round_5(self, message):
        return self._round(5, message)
