"""Pins the oracle against the reference's own routines (translated, oracle/_ref; see test_oracle_vs_reference.py and
test_oracle_vs_reference_smoothers.py) in the flow regimes of tests/regimes.py, where the sensor cap, the supersonic
far-field branches, the pressure floors and the SA rr clip are taken.  Bit-exact.  Skips when the library was not built."""
import numpy as np
import pytest

import regimes as R
from oracle import refblockette as rb
from test_oracle_vs_reference import DISCS, DISS_APPROX, FLOW, TURB, VISC_APPROX, _compare_dw
from test_oracle_vs_reference_bcs import _check
from test_oracle_vs_reference_smoothers import _eq, _oracle

pytestmark = pytest.mark.skipif(not rb.available(), reason="oracle/_ref/libblockette_ref.so not built")

SHAPE = (12, 10, 8)


def _prepared(regime, options, shape=SHAPE):
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case(regime, shape, options)
    Oracle(hb, prm).reference_shock_sensor()    # input of the approximate-dissipation paths
    return prm, hb


@pytest.mark.parametrize("regime", R.REGIMES)
@pytest.mark.parametrize("eq", ["Euler", "laminar NS", "RANS"])
@pytest.mark.parametrize("disc", DISCS)
def test_residual_core_in_regimes(regime, eq, disc):
    prm, hb = _prepared(regime, {"equationType": eq, "discretization": disc})
    _compare_dw(prm, hb, FLOW | TURB)


# Unlimited second-order states across a density jump of 8 are negative in places and the Roe flux is NaN -- in the
# reference's inviscidUpwindFlux as much as in the oracle (checked bit for bit, NaN included); "no limiter" is therefore
# pinned on the regimes without such a jump only.
JUMP_REGIMES = ("contact_i", "contact_j", "contact_k", "contact_pocket", "supersonic")
LIMITER_CASES = [(r, lim) for r in R.REGIMES for lim in ("first order", "no limiter", "van Albada", "minmod")
                 if not (lim == "no limiter" and r in JUMP_REGIMES)]


@pytest.mark.parametrize("regime,limiter", LIMITER_CASES)
def test_upwind_limiters_in_regimes(regime, limiter):
    prm, hb = _prepared(regime, {"equationType": "RANS", "discretization": "upwind", "limiter": limiter})
    _compare_dw(prm, hb, FLOW | TURB)


@pytest.mark.parametrize("regime", R.REGIMES)
@pytest.mark.parametrize("disc", DISCS)
@pytest.mark.parametrize("flags", [DISS_APPROX, VISC_APPROX, DISS_APPROX | VISC_APPROX])
def test_approximate_paths_in_regimes(regime, disc, flags):
    """*Approx routines of the ANK/NK preconditioner assembly; the frozen sensor of the approximate dissipation is
    capped in the contact, supersonic and floor regimes"""
    prm, hb = _prepared(regime, {"equationType": "RANS", "discretization": disc})
    _compare_dw(prm, hb, FLOW | TURB | flags)


@pytest.mark.parametrize("regime", ["supersonic", "low_mach", "floors", "contact_k"])
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
def test_bcs_in_regimes(regime, eq):
    prm, hb = R.regime_case(regime, (9, 8, 7), {"equationType": eq})
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    _check(prm, hb, True)
    _check(prm, hb, False)


@pytest.mark.parametrize("regime", ["supersonic", "low_mach", "stagnation"])
def test_turbulence_bcs_in_regimes(regime):
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case(regime, (9, 8, 7), {"equationType": "RANS"})
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    ho = hb.copy()
    Oracle(ho, prm).apply_turb_bc(True)
    rb.call(hb, prm, "turbbcroutines_bcturbtreatment")
    r = rb.again("turbbcroutines_applyallturbbcthisblock", 1)
    _eq(r.a["w"][..., 5], ho.w[..., 5], "nuTilde halos")
    _eq(r.a["rev"], ho.rev, "rev")


# ---------------------------------------------------------------------------------------------------------------------
# smoother stages
SMOOTHER_REGIMES = ["contact_i", "contact_pocket", "supersonic", "low_mach", "stagnation", "floors"]


def _residual_state(regime, options, shape=SHAPE):
    """block with a freshly computed residual, time step and spectral radii (what the smoothers see)"""
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case(regime, shape, options)
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    o = Oracle(hb, prm)
    o.time_step(True)
    o.residual_block(1.0)
    hb.wn[...] = hb.w[..., :5]
    hb.pn[...] = hb.p
    return prm, hb


@pytest.mark.parametrize("regime", SMOOTHER_REGIMES)
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
@pytest.mark.parametrize("stage,avg", [(1, "never"), (2, "alternate"), (5, "never")])
def test_rk_stage_in_regimes(regime, eq, stage, avg):
    prm, hb = _residual_state(regime, {"equationType": eq, "resAveraging": avg})
    ho, o = _oracle(hb, prm)
    o.rk_stage(stage)
    r = rb.call(hb, prm, "smoothers_executerkstage", rkstage=stage)
    for l in range(5):
        _eq(r.a["w"][..., l], ho.w[..., l], "w[%d]" % l)
    _eq(r.a["p"], ho.p, "p")
    _eq(r.a["rlv"], ho.rlv, "rlv")
    _eq(r.a["rev"], ho.rev, "rev")


def test_rk_stage_density_and_pressure_floors():
    """a stage of a boundary-spanning contact drives cells through the update's floors 1e-4 rhoInf and 1e-4 pInfCorr
    (executeRkStage, smoothers.F90:90-382); the oracle floors them as the reference does"""
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case("contact_k", (16, 12, 10), {"equationType": "Euler", "resAveraging": "never"})
    o = Oracle(hb, prm)
    o.apply_flow_bc(True)
    o.time_step(True)
    o.residual_block(1.0)
    hb.wn[...] = hb.w[..., :5]
    hb.pn[...] = hb.p
    ho, o = _oracle(hb, prm)
    o.rk_stage(1)
    r = rb.call(hb, prm, "smoothers_executerkstage", rkstage=1)
    ow = hb.d.owned()
    assert (ho.w[ow + (0,)] == R.PRESSURE_FLOOR * prm.rhoInf).any()
    assert (ho.p[ow] == R.PRESSURE_FLOOR * prm.pInfCorr).any()
    _eq(r.a["w"], ho.w, "w")
    _eq(r.a["p"], ho.p, "p")


@pytest.mark.parametrize("regime", ["contact_pocket", "supersonic", "low_mach", "stagnation"])
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
def test_full_runge_kutta_cycle_in_regimes(regime, eq):
    from oracle.pyoracle import Oracle

    prm, hb = _residual_state(regime, {"equationType": eq})
    hb.fw[...] = 0.0
    Oracle(hb, prm).residual_block(prm.cdisRK[0])
    ho, o = _oracle(hb, prm)
    o.rk_smoother()
    r = rb.call(hb, prm, "smoothers_rungekuttasmoother")
    ow = hb.d.owned()
    assert np.isfinite(ho.w[ow]).all()
    for l in range(5):
        _eq(r.a["w"][..., l], ho.w[..., l], "w[%d]" % l)
    _eq(r.a["p"], ho.p, "p")


@pytest.mark.parametrize("regime", SMOOTHER_REGIMES)
def test_residual_averaging_in_regimes(regime):
    prm, hb = _residual_state(regime, {"equationType": "RANS", "resAveraging": "always"})
    ho, o = _oracle(hb, prm)
    o.residual_averaging()
    r = rb.call(hb, prm, "residuals_residualaveraging")
    ow = hb.d.owned()
    _eq(r.a["dw"][ow][..., :5], ho.dw[ow][..., :5], "dw")


@pytest.mark.parametrize("regime", SMOOTHER_REGIMES)
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
def test_compute_dw_dadi_in_regimes(regime, eq):
    prm, hb = _residual_state(regime, {"equationType": eq})
    ow = hb.d.owned()
    hb.dw[ow + (slice(0, 5),)] *= (-prm.cfl * hb.dtl[ow] * hb.vol[ow])[..., None]
    ho, o = _oracle(hb, prm)
    o.compute_dw_dadi()
    r = rb.call(hb, prm, "residuals_computedwdadi")
    for l in range(5):
        _eq(r.a["dw"][ow][..., l], ho.dw[ow][..., l], "dw[%d]" % l)


@pytest.mark.parametrize("regime", SMOOTHER_REGIMES)
@pytest.mark.parametrize("eq,avg", [("Euler", "never"), ("RANS", "never"), ("RANS", "always")])
def test_dadi_step_in_regimes(regime, eq, avg):
    prm, hb = _residual_state(regime, {"equationType": eq, "resAveraging": avg, "smoother": "DADI"})
    ho, o = _oracle(hb, prm)
    o.dadi_step()
    r = rb.call(hb, prm, "smoothers_executedadistep", rkstage=0)
    for l in range(5):
        _eq(r.a["w"][..., l], ho.w[..., l], "w[%d]" % l)
    _eq(r.a["p"], ho.p, "p")


@pytest.mark.parametrize("regime", ["stagnation", "supersonic", "contact_pocket", "low_mach", "floors"])
def test_sa_block_in_regimes(regime):
    """sa_block (src/turbulence/sa.F90:16-86) incl. the DD-ADI solve; stagnation reaches the rr clip of saSource"""
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case(regime, SHAPE, {"equationType": "RANS"})
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    ho = hb.copy()
    Oracle(ho, prm).sa_block()
    r = rb.call(hb, prm, "sa_sa_block", 0)
    ow = hb.d.owned()
    _eq(r.a["dw"][ow][..., 5], ho.dw[ow][..., 5], "dw(itu1)")
    _eq(r.a["w"][..., 5], ho.w[..., 5], "nuTilde (whole box)")
    _eq(r.a["rev"], ho.rev, "rev")
