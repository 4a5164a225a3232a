"""Helpers the oracle's CPU tests share."""
import pytest

from oracle import plonk_oracle as O


@pytest.fixture
def host_lincomb(monkeypatch):
    """the product's host verifier with its G1 combinations by the oracle's double-and-add (the CPU tests have no GPU);
    returns the plonkathon_b200 package"""
    import plonkathon_b200 as pb
    from plonkathon_b200 import verifier

    def lincomb(pairs, ctx=None):
        live = [((int(p[0]), int(p[1])), int(k) % O.R_MOD) for p, k in pairs if p is not None]
        res = O.ec_lincomb_naive(live)
        return None if res is None else (pb.FQ(res[0]), pb.FQ(res[1]))
    monkeypatch.setattr(verifier, "ec_lincomb", lincomb)
    return pb
