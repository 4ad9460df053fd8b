"""The restatement of infChangeCorrection and setUniformFlow in tests/inf_change.py, which the GPU tests hold the device
to: its skip rule, its rotation, its invariants and the reference details it keeps (the stale pressure of the BC halos,
NaN from "rotate" with a change of speed alone)."""
import math

import numpy as np
import pytest

import inf_change as IC
from util import MIXED, case

EQS = ["Euler", "laminar NS", "RANS"]
EPS = np.finfo(float).eps


def _old(prm):
    return list(prm.wInf)[:5]


@pytest.mark.parametrize("change,lift", [("alpha", 2), ("alpha", 3), ("mach", 2), ("pressure", 2), ("temperature", 2)])
def test_free_stream_pairs_change_the_measured_part(change, lift):
    prm0, prm1 = IC.free_stream_pair("RANS", change, lift)
    d = IC.delta_winf(prm1, _old(prm0))
    assert IC.my_norm2(d) > 1e-4   # far above the default tolerance of 1e-12
    assert prm1.wInf[5] == prm0.wInf[5]
    same = IC.with_free_stream(prm0, 0.8, 1.8, lift)
    assert list(same.wInf) == list(prm0.wInf) and same.pInfCorr == prm0.pInfCorr and same.rhoInf == prm0.rhoInf


def test_skip_rule_measures_rho_u_v_only():
    """myNorm2 takes a dimension(3) dummy: alpha +2 -> -2 degrees with liftIndex 3 changes w alone and is skipped"""
    prm0, prm1 = IC.sign_flip_pair("RANS")
    d = IC.delta_winf(prm1, _old(prm0))
    assert d[0] == d[1] == d[2] == 0.0 and d[3] != 0.0
    assert IC.skipped(prm1, _old(prm0), 1e-12)
    assert IC.skipped(prm0, _old(prm0), 1e-12)
    prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
    n = IC.my_norm2(IC.delta_winf(prm1, _old(prm0)))
    assert IC.skipped(prm1, _old(prm0), np.nextafter(n, np.inf))
    assert not IC.skipped(prm1, _old(prm0), n)
    hb = case(8, 7, 6)[1]
    ref = hb.copy()
    assert not IC.inf_change_correction([ref], prm1, _old(prm0), tol=np.nextafter(n, np.inf))
    assert np.array_equal(ref.w, hb.w)


@pytest.mark.parametrize("lift", [2, 3])
def test_rotation_matrix(lift):
    prm0, prm1 = IC.free_stream_pair("RANS", "alpha", lift)
    v1, v2 = _old(prm0)[1:4], list(prm1.wInf)[1:4]
    R = np.array(IC.rot_matrix(v1, v2))
    assert np.abs(R @ R.T - np.eye(3)).max() < 8 * EPS
    r = R @ np.array(v1) * (IC.my_norm2(v2) / IC.my_norm2(v1))
    assert np.abs(r - np.array(v2)).max() < 1e-14 * IC.my_norm2(v2)


@pytest.mark.parametrize("change", ["mach", "pressure"])
def test_rotate_without_a_change_of_direction_is_not_finite(change):
    """a change of speed alone: vec1 x vec2 = 0 and the reference normalises 0 / 0, so every velocity becomes NaN.  This is
    why the device refuses "rotate" here instead of writing that state."""
    prm0, prm1 = IC.free_stream_pair("RANS", change, 2)
    assert not np.isfinite(IC.rot_matrix(_old(prm0)[1:4], list(prm1.wInf)[1:4])).all()
    hb = case(8, 7, 6)[1]
    IC.correct_owned(hb, prm1, _old(prm0), "rotate")
    ow = hb.d.owned()
    assert np.isnan(hb.w[ow + (1,)]).all() and np.isfinite(hb.w[ow + (0,)]).all()


@pytest.mark.parametrize("kind", IC.KINDS)
@pytest.mark.parametrize("lift", [2, 3])
@pytest.mark.parametrize("eq", EQS)
def test_uniform_old_free_stream_becomes_the_new_one(eq, lift, kind):
    """offset is exact; rotate is exact in rho and rho E, and the velocity follows to the conditioning of the reference's
    acos near 1: an error of one rounding in the cosine moves the angle by eps / sin(theta), 6e-15 for one degree"""
    prm0, prm1 = IC.free_stream_pair(eq, "alpha", lift)
    hb = case(8, 7, 6, IC.options(eq, lift))[1]
    hb.w[...] = np.asarray(prm0.wInf[:hb.nw])
    IC.correct_owned(hb, prm1, _old(prm0), kind)
    ow = hb.d.owned()
    speed = IC.my_norm2(list(prm1.wInf)[1:4])
    theta = math.radians(1.0)
    for l in range(5):
        err = np.abs(hb.w[ow + (l,)] - prm1.wInf[l]).max()
        if kind == "offset" or l in (0, 4):
            assert err <= 1e-15 * abs(prm1.wInf[l]), (l, err)
        else:
            assert err <= 4 * EPS / math.sin(theta) * speed, (l, err / speed)
    if hb.nw == 6:
        assert np.all(hb.w[ow + (5,)] == prm0.wInf[5])   # the turbulence variable is not corrected


@pytest.mark.parametrize("split", [None, MIXED])
def test_boundary_halos_use_the_pressure_as_it_was(split):
    """the reference applies the flow BCs to the corrected w without recomputing p: halos differ from those built on the
    pressure of the corrected state, and the owned pressure is not changed"""
    from oracle.pyoracle import Oracle

    prm0, prm1 = IC.free_stream_pair("RANS", "mach", 2)
    hb = case(9, 8, 7, split=split)[1]
    stale = hb.copy()
    IC.inf_change_correction([stale], prm1, _old(prm0))
    ow = hb.d.owned()
    assert np.array_equal(stale.p[ow], hb.p[ow])
    fresh = hb.copy()
    IC.correct_owned(fresh, prm1, _old(prm0), "offset")
    Oracle(fresh, prm1).pressure(False)
    Oracle(fresh, prm1).apply_flow_bc(True)
    assert np.abs(fresh.w - stale.w).max() > 0


@pytest.mark.parametrize("eq", EQS)
def test_set_uniform_flow_on_levels_1_and_2(eq):
    from adflow_b200 import synthetic as syn

    prm, hb = case(12, 10, 8, IC.options(eq, 2))
    coarse = syn.make_coarse_block(hb, prm)
    mu, ratio = 1.7e-3, 0.009
    for blk in (hb, coarse):
        b = blk.copy()
        b.dw[...] = 1.0; b.fw[...] = 1.0; b.rlv[...] = 2.0; b.rev[...] = 3.0
        IC.set_uniform_flow(b, prm, mu, ratio)
        assert np.all(b.w == np.asarray(prm.wInf[:b.nw])) and not b.dw.any() and not b.fw.any()
        assert np.all(b.p == prm.pInfCorr)
        assert np.all(b.rlv == (2.0 if eq == "Euler" else mu))
        assert np.all(b.rev == (ratio * mu if eq == "RANS" else 3.0))
