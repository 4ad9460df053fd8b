"""The regime generator (tests/regimes.py) reaches the branches it is meant to reach, and its numpy sensors are the
oracle's.  Runs without a GPU and without the reference."""
import numpy as np
import pytest

import regimes as R
from util import FLOW, TURB, case, oracle_residual

SHAPE = (12, 10, 8)

# branch counts every regime must keep > 0 (RANS, scalar dissipation unless stated)
EXPECT = {
    "contact_i": ["sensor_cap_i", "dis4_zero_i"],
    "contact_j": ["sensor_cap_j", "dis4_zero_j"],
    "contact_k": ["sensor_cap_k", "dis4_zero_k"],
    "contact_pocket": ["sensor_cap_i", "sensor_cap_j", "sensor_cap_k"],
    "supersonic": ["sensor_cap_i", "sensor_cap_j", "sensor_cap_k", "matrix_sensor_cap_i", "matrix_sensor_cap_j",
                   "matrix_sensor_cap_k", "supersonic_i", "ff_sup_in", "ff_sup_out", "ff_sub_in", "ff_sub_out"],
    "stagnation": ["stagnant_i", "stagnant_j", "stagnant_k", "sa_rr_clip"],
    "floors": ["p_floor", "turb_clip", "sensor_cap_i", "matrix_sensor_cap_i"],
    "low_mach": ["ff_sub_in", "ff_sub_out"],
    "low_reynolds": ["low_cell_re"],
}


def assert_reaches(prm, hb, regime, keys=None):
    r = R.reach(prm, hb, regime)
    missing = [k for k in (EXPECT[regime] if keys is None else keys) if r.get(k, 0) <= 0]
    assert not missing, "regime %s no longer reaches %s: %s" % (regime, missing, r)
    return r


@pytest.mark.parametrize("regime", R.REGIMES)
def test_regime_reaches_its_branches(regime):
    prm, hb = R.regime_case(regime, SHAPE)
    assert_reaches(prm, hb, regime)
    assert np.isfinite(hb.w).all() and (hb.p > 0).all() and (hb.w[..., 0] > 0).all()


def test_smooth_state_reaches_none_of_them():
    """the default synthetic state takes none of these branches: the regimes are what exercises them"""
    smooth = R.reach(*case(*SHAPE))
    for k in ("sensor_cap_i", "sensor_cap_j", "sensor_cap_k", "ff_sup_in", "ff_sup_out", "p_floor", "turb_clip", "sa_rr_clip"):
        assert smooth[k] == 0, k


@pytest.mark.parametrize("eq", ["RANS", "laminar NS"])
def test_low_reynolds_cells_only_at_low_pressure(eq):
    """at 20 kPa no owned cell is viscous-dominated; at the low_reynolds regime's 2 Pa every one is"""
    assert R.reach(*case(*SHAPE, {"equationType": eq}))["low_cell_re"] == 0
    prm, hb = R.regime_case("low_reynolds", SHAPE, {"equationType": eq})
    assert R.reach(prm, hb)["low_cell_re"] == hb.d.nx * hb.d.ny * hb.d.nz


def test_low_mach_far_field_in_and_out_on_both_j_faces():
    prm, hb = R.regime_case("low_mach", SHAPE)
    _, byface = R.farfield_branches(prm, hb)
    assert byface[R.syn.JMIN]["ff_sub_in"] > 0 and byface[R.syn.JMAX]["ff_sub_out"] > 0


def test_supersonic_far_field_sides():
    prm, hb = R.regime_case("supersonic", SHAPE)
    _, byface = R.farfield_branches(prm, hb)
    assert byface[R.syn.IMIN]["ff_sup_in"] > 0 and byface[R.syn.IMAX]["ff_sup_out"] > 0


@pytest.mark.parametrize("regime", ["contact_i", "contact_j", "contact_k", "contact_pocket", "supersonic", "floors"])
@pytest.mark.parametrize("eq", ["RANS", "Euler"])
def test_numpy_entropy_sensor_is_the_oracles(regime, eq):
    """entropy_sensor (numpy) against the dss the oracle's scalar dissipation stores (cells 1..ie)"""
    prm, hb = R.regime_case(regime, SHAPE, {"equationType": eq})
    ho = oracle_residual(prm, hb, FLOW | TURB if eq == "RANS" else FLOW)
    d = hb.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    mine = R.entropy_sensor(prm, hb)[c1]
    assert np.abs(mine - ho.dss[c1]).max() < 1e-12 * max(1.0, np.abs(ho.dss[c1]).max())
    assert ho.dss[c1].max() > 0.25 or eq == "Euler"


@pytest.mark.parametrize("regime", ["supersonic", "floors"])
def test_numpy_pressure_sensor_is_the_oracles(regime):
    """pressure_sensor (numpy) against the dss the oracle's matrix dissipation stores"""
    prm, hb = R.regime_case(regime, SHAPE, {"discretization": "central plus matrix dissipation"})
    ho = oracle_residual(prm, hb, FLOW | TURB)
    d = hb.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    mine = R.pressure_sensor(prm, hb)[c1]
    assert np.abs(mine - ho.dss[c1]).max() < 1e-12
    assert ho.dss[c1].max() > 0.25
