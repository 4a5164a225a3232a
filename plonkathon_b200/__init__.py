"""plonkathon_b200 -- H100-native PLONK/KZG proving hot path behind the reference's Python surface
(0xPARC/plonkathon: curve.py, poly.py, setup.py, prover.py, transcript.py, verifier.py)."""
from .field import FQ, FQ2, CURVE_ORDER, FIELD_MODULUS  # noqa: F401
from .curve import (Scalar, ec_lincomb, ec_mul, G1Point, G2Point, G1, G2, g2_add, g2_mul,  # noqa: F401
                    pairing_product_is_one)
from .poly import Basis, Polynomial  # noqa: F401
from .setup import Setup  # noqa: F401
from .verifier import VerificationKey  # noqa: F401
from ._lib import Context, PlonkB200Error, default_context  # noqa: F401
from .transcript import Transcript, Message1, Message2, Message3, Message4, Message5  # noqa: F401
from .prover import Prover, Proof, LookupProof, NextRowProof, ShuffleProof, NextRowShuffleProof  # noqa: F401
from .wiring import permutation_arrays  # noqa: F401
from .witness import WitnessReport  # noqa: F401
from .solve import WireSolution, solve_wires  # noqa: F401
