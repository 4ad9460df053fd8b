"""The restatement of tests/inf_change.py, which the GPU tests hold the device to, against the reference's own
infChangeCorrection, setUniformFlow and getRotMatrix (translated, tests/ref_inf_change.py), bit for bit on the whole box,
halos included.  On one block the reference's whalo2 exchanges nothing and ends with computeEtotBlock on the owned cells,
so the comparison covers the owned-cell update, the flow BCs from the corrected w and the old pressure, the total energy
formed from that old pressure, and with oversetPresent the turbulence and flow BCs applied again.  The reference side
skips when the reference source or oracle/_ref is absent."""
import numpy as np
import pytest

import inf_change as IC
import ref_inf_change as R
from util import MIXED, case

needs_ref = pytest.mark.skipif(not R.available(), reason="reference source or oracle/_ref/libblockette_ref.so not present")
EQS = ["Euler", "laminar NS", "RANS"]
CHANGES = [("alpha", 2, "offset"), ("alpha", 2, "rotate"), ("alpha", 3, "offset"), ("alpha", 3, "rotate"),
           ("mach", 2, "offset"), ("pressure", 2, "offset"), ("temperature", 2, "offset")]


def _old(prm):
    return list(prm.wInf)[:5]


def _eq(a, b, what):
    assert np.array_equal(a, b, equal_nan=True), "%s differs: max abs %.3e" % (what, np.nanmax(np.abs(a - b)))


def _same_state(a, b, fields=("w", "p", "rlv", "rev")):
    for f in fields:
        _eq(getattr(a, f), getattr(b, f), f)


@needs_ref
@pytest.mark.parametrize("layout", ["default", "MIXED"])
@pytest.mark.parametrize("change,lift,kind", CHANGES, ids=["%s-lift%d-%s" % c for c in CHANGES])
@pytest.mark.parametrize("eq", EQS)
def test_correction(eq, change, lift, kind, layout):
    prm0, prm1 = IC.free_stream_pair(eq, change, lift)
    hb = case(11, 9, 10, IC.options(eq, lift), split=MIXED if layout == "MIXED" else None)[1]
    mine, ref = hb.copy(), hb.copy()
    assert IC.inf_change_correction([mine], prm1, _old(prm0), kind=kind)
    R.inf_change_correction(ref, prm1, _old(prm0), kind=kind)
    assert np.abs(ref.w - hb.w).max() > 0
    _same_state(mine, ref)


@needs_ref
@pytest.mark.parametrize("kind", IC.KINDS)
@pytest.mark.parametrize("eq", ["laminar NS", "RANS"])
def test_correction_with_overset_present(eq, kind):
    """oversetPresent: the turbulence (RANS) and flow BCs once more after whalo2"""
    prm0, prm1 = IC.free_stream_pair(eq, "alpha", 2)
    hb = case(10, 9, 8, IC.options(eq, 2))[1]
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)  # the reference numbers viscous subfaces first
    mine, ref = hb.copy(), hb.copy()
    IC.inf_change_correction([mine], prm1, _old(prm0), kind=kind, overset=True)
    R.inf_change_correction(ref, prm1, _old(prm0), kind=kind, overset=True)
    _same_state(mine, ref)
    plain = hb.copy()
    IC.inf_change_correction([plain], prm1, _old(prm0), kind=kind)
    assert np.abs(plain.w - ref.w).max() > 0


def _skip_cases():
    prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
    n = IC.my_norm2(IC.delta_winf(prm1, _old(prm0)))
    flip0, flip1 = IC.sign_flip_pair("RANS")
    return {"identical": (prm0, prm0, 1e-12, True), "lift3-sign-flip": (flip0, flip1, 1e-12, True),
            "tol-just-above": (prm0, prm1, np.nextafter(n, np.inf), True), "tol-at-the-change": (prm0, prm1, n, False),
            "tol-just-below": (prm0, prm1, np.nextafter(n, 0.0), False)}


@needs_ref
@pytest.mark.parametrize("name", list(_skip_cases()))
@pytest.mark.parametrize("kind", IC.KINDS)
def test_skip_rule(name, kind):
    prm0, prm1, tol, skip = _skip_cases()[name]
    hb = case(9, 8, 7, IC.options("RANS", 3 if "lift3" in name else 2))[1]
    mine, ref = hb.copy(), hb.copy()
    assert IC.inf_change_correction([mine], prm1, _old(prm0), tol=tol, kind=kind) == (not skip)
    R.inf_change_correction(ref, prm1, _old(prm0), tol=tol, kind=kind)
    _same_state(mine, ref)
    if skip:
        _same_state(ref, hb)


@needs_ref
@pytest.mark.parametrize("change", ["mach", "pressure"])
def test_rotate_with_a_change_of_speed_alone_gives_non_finite_velocities(change):
    """the reason the device refuses it"""
    prm0, prm1 = IC.free_stream_pair("RANS", change, 2)
    ref = case(9, 8, 7)[1]
    R.inf_change_correction(ref, prm1, _old(prm0), kind="rotate")
    ow = ref.d.owned()
    for l in (1, 2, 3):
        assert not np.isfinite(ref.w[ow + (l,)]).any()
    assert not np.isfinite(R.rot_matrix(_old(prm0)[1:4], list(prm1.wInf)[1:4])).all()


@needs_ref
@pytest.mark.parametrize("vecs", [((1.0, 0.03, 0.0), (1.0, 0.05, 0.0)), ((0.9, 0.02, 0.03), (0.95, -0.01, 0.04)),
                                  ((0.8, 0.0, 0.02), (0.8, 0.0, -0.02))])
def test_rotation_matrix(vecs):
    assert R.rot_matrix(*vecs) == IC.rot_matrix(*vecs)


@needs_ref
@pytest.mark.parametrize("level", [1, 2])
@pytest.mark.parametrize("eq", EQS)
def test_set_uniform_flow(eq, level):
    """on a level-1 block and, as mgStartLevel = 2, on a level-2 block bound with its own arrays"""
    from adflow_b200 import synthetic as syn

    prm, hb = case(12, 10, 8, IC.options(eq, 2))
    blk = hb if level == 1 else syn.make_coarse_block(hb, prm)
    blk.dw[...] = 1.0; blk.fw[...] = 1.0
    mine, ref = blk.copy(), blk.copy()
    mu, ratio = 1.7e-3, 0.009
    IC.set_uniform_flow(mine, prm, mu, ratio)
    R.set_uniform_flow(ref, prm, mu, ratio, level)
    _same_state(mine, ref, ("w", "p", "rlv", "rev", "dw", "fw"))
