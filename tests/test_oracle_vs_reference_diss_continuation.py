"""Dissipation-based continuation: the oracle with the coefficients of tests/diss_continuation.py against the reference's
own routines (translated, oracle/_ref) with useDissContinuation, dissContMagnitude/Midpoint/Sharpness and
iteration%totalR / totalR0 set, bit for bit; that the flow regimes the GPU tests use make the continuation term large;
and getFreeStreamResidual composed from oracle routines.  The reference side skips when its library was not built."""
import numpy as np
import pytest

import diss_continuation as DC
import regimes as R
from oracle import refblockette as rb
from util import case

FLOW, TURB, INTERMED, DISS_APPROX = 8, 16, 4, 1
needs_ref = pytest.mark.skipif(not rb.available(), reason="oracle/_ref/libblockette_ref.so not built")


@pytest.fixture
def ref_totals(monkeypatch):
    """the translated reference with the continuation options of the parameters and the given totals"""
    state = {}
    original = rb.set_params

    def set_params(prm, nw, rfil=1.0):
        original(prm, nw, rfil)
        rb._seti("usedisscontinuation", prm.useDissContinuation)
        for n in ("dissContMagnitude", "dissContMidpoint", "dissContSharpness"):
            rb._setd(n.lower(), getattr(prm, n))
        rb._setd("totalr", state["totalR"]); rb._setd("totalr0", state["totalR0"])

    monkeypatch.setattr(rb, "set_params", set_params)

    def use(total_r, total_r0):
        state["totalR"], state["totalR0"] = total_r, total_r0

    return use


def _eq(a, b, what):
    assert np.array_equal(a, b, equal_nan=True), "%s differs: max abs %.3e" % (what, np.nanmax(np.abs(a - b)))


def _prepared(options, shape=(11, 9, 10), regime=None):
    from oracle.pyoracle import Oracle

    opt = dict(DC.OPTIONS, **options)
    prm, hb = R.regime_case(regime, shape, opt) if regime else case(*shape, opt)
    Oracle(hb, prm).reference_shock_sensor()   # input of the approximate dissipation
    return prm, hb


def _oracle_core(prm, hb, flags, rfil=1.0):
    from oracle.pyoracle import Oracle

    ho = hb.copy()
    Oracle(ho, prm).residual_core(flags, rfil)
    return ho


# ---------------------------------------------------------------------------------------------------------------------
def test_coefficients():
    prm = case(4, 4, 4, DC.OPTIONS)[0]
    v, m = prm.vis2, prm.dissContMagnitude
    assert DC.coef(prm, 1.0, 1.0) == v + m / (1 + np.exp(-9.0))
    assert DC.coef(prm, 0.0, 1.0) == DC.coef(prm, 1.0, 0.0) == DC.coef(prm, 0.0, 0.0) == DC.coef(prm, 1.0, 1.0)
    assert abs(DC.coef(prm, 1e-8, 1.0) - v) < 1e-6 * m
    assert DC.coef_approx(prm, 0.0, 1.0) == v
    assert np.isnan(DC.coef_approx(prm, 0.0, 0.0))
    assert DC.coef_approx(prm, 1.0, 0.0) == v + m
    assert DC.coef(DC.plain(prm), 1e-3, 1.0) == DC.coef_approx(DC.plain(prm), 0.0, 0.0) == v


@needs_ref
@pytest.mark.parametrize("totals", DC.TOTALS)
@pytest.mark.parametrize("eq", ["Euler", "laminar NS", "RANS"])
def test_residual_core(ref_totals, eq, totals):
    prm, hb = _prepared({"equationType": eq}, regime="supersonic")
    ref_totals(*totals)
    ho = _oracle_core(DC.oracle_params(prm, *totals), hb, FLOW | TURB)
    r = rb.residual_core(hb, prm, FLOW | TURB)
    ow = hb.d.owned()
    for l in range(hb.nw):
        _eq(r.a["dw"][ow + (l,)], ho.dw[ow + (l,)], "dw[%d]" % l)


@needs_ref
@pytest.mark.parametrize("totals", DC.TOTALS + [(0.0, 0.0)])
def test_approximate_residual(ref_totals, totals):
    """inviscidDissFluxScalarApprox: no zero guard (totalR = 0 gives vis2, both zero NaN, in the reference as here)"""
    prm, hb = _prepared({"equationType": "RANS"}, regime="supersonic")
    ref_totals(*totals)
    ho = _oracle_core(DC.oracle_params(prm, *totals, approx=True), hb, FLOW | TURB | DISS_APPROX)
    r = rb.residual_core(hb, prm, FLOW | TURB | DISS_APPROX)
    ow = hb.d.owned()
    for l in range(5):
        _eq(r.a["dw"][ow + (l,)], ho.dw[ow + (l,)], "dw[%d]" % l)
    assert np.isnan(ho.dw[ow + (0,)]).all() == (totals == (0.0, 0.0))


@needs_ref
@pytest.mark.parametrize("totals", DC.TOTALS[:3])
@pytest.mark.parametrize("rfil", [1.0, 0.56, 0.44])
def test_residual_at_runge_kutta_fractions(ref_totals, rfil, totals):
    prm, hb = _prepared({"equationType": "RANS"}, regime="contact_pocket")
    ref_totals(*totals)
    ho = _oracle_core(DC.oracle_params(prm, *totals), hb, FLOW | TURB, rfil)
    r = rb.residual_core(hb, prm, FLOW | TURB, rfil)
    ow = hb.d.owned()
    for l in range(5):
        _eq(r.a["dw"][ow + (l,)], ho.dw[ow + (l,)], "dw[%d]" % l)


def _smoother_state(totals, options, regime="contact_pocket"):
    """block with residual, time step and radii from the oracle with continuation (what the smoothers see)"""
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case(regime, (12, 9, 10), dict(DC.OPTIONS, **options))
    o = Oracle(hb, DC.oracle_params(prm, *totals))
    o.time_step(True)
    o.residual_block(1.0)
    hb.wn[...] = hb.w[..., :5]
    hb.pn[...] = hb.p
    return prm, hb


@needs_ref
@pytest.mark.parametrize("totals", [DC.TOTALS[1], DC.TOTALS[3]])
@pytest.mark.parametrize("stage", [2, 4])
def test_rk_stage(ref_totals, stage, totals):
    """executeRkStage: residual_block at rFil = cdisRK(stage + 1) = 0.56 / 0.44 with the block flux routines of fluxes.F90"""
    from oracle.pyoracle import Oracle

    prm, hb = _smoother_state(totals, {"equationType": "RANS"})
    assert prm.cdisRK[stage] in (0.56, 0.44)
    ref_totals(*totals)
    ho = hb.copy()
    Oracle(ho, DC.oracle_params(prm, *totals)).rk_stage(stage)
    r = rb.call(hb, prm, "smoothers_executerkstage", rkstage=stage)
    for l in range(5):
        _eq(r.a["w"][..., l], ho.w[..., l], "w[%d]" % l)
    _eq(r.a["p"], ho.p, "p")


@needs_ref
@pytest.mark.parametrize("totals", [DC.TOTALS[1], DC.TOTALS[4]])
def test_dadi_step(ref_totals, totals):
    from oracle.pyoracle import Oracle

    prm, hb = _smoother_state(totals, {"equationType": "RANS", "smoother": "DADI"})
    ref_totals(*totals)
    ho = hb.copy()
    Oracle(ho, DC.oracle_params(prm, *totals)).dadi_step()
    r = rb.call(hb, prm, "smoothers_executedadistep", rkstage=0)
    for l in range(5):
        _eq(r.a["w"][..., l], ho.w[..., l], "w[%d]" % l)
    _eq(r.a["p"], ho.p, "p")


# ---------------------------------------------------------------------------------------------------------------------
# reach: where the GPU tests hold the device to 1e-12 (rel L2 of a row), the continuation term has to be far larger
REACH = [("supersonic", "RANS"), ("supersonic", "Euler"), ("contact_pocket", "RANS"), ("contact_k", "laminar NS"),
         ("stagnation", "RANS")]


@pytest.mark.parametrize("regime,eq", REACH)
def test_continuation_term_is_large_in_the_gpu_states(regime, eq):
    from util import rel_l2

    prm, hb = _prepared({"equationType": eq}, shape=(12, 10, 8), regime=regime)
    flags = FLOW | (TURB if eq == "RANS" else 0)
    for totals in DC.TOTALS[:2]:
        on = _oracle_core(DC.oracle_params(prm, *totals), hb, flags)
        off = _oracle_core(DC.plain(prm), hb, flags)
        ow = hb.d.owned()
        for l in range(5):
            assert rel_l2(on.dw[ow + (l,)], off.dw[ow + (l,)]) > 1e3 * 1e-12, (regime, eq, totals, l)


# ---------------------------------------------------------------------------------------------------------------------
# getFreeStreamResidual (NKSolvers.F90:280-333), composed from oracle routines: w = wInf on the whole box, blocketteRes
# with useUpdateIntermed (p, rlv, rev, BCs, whalo2's owned-cell etot, core), the sums of getCurrentResidual
def _free_stream_prepared(prm, hb):
    """w = wInf on the whole box, then the preamble of blocketteRes: p, rlv, rev, BCs, whalo2's owned-cell etot"""
    import ctypes as C

    from oracle.pyoracle import Oracle

    h2 = hb.copy()
    h2.w[...] = np.asarray(prm.wInf[:hb.nw])
    o = Oracle(h2, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    return h2


def oracle_free_stream_residual(prm, hb):
    """(sum (dw_rho / vol)^2, sum (dw / vol)^2 with turbResScale on the turbulence row) of the uniform free stream,
    and the block it was evaluated on"""
    from oracle.pyoracle import Oracle

    h2 = _free_stream_prepared(prm, hb)
    o = Oracle(h2, prm)
    o.residual_core(FLOW | TURB | INTERMED)
    return o.norms(), h2


@needs_ref
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
def test_free_stream_residual_composition_matches_reference(ref_totals, eq):
    """the core of that composition in the reference's blocketteResCore, with continuation at the library's initial
    totals (0, 0); the preamble and the sums are pinned by the existing oracle-vs-reference tests"""
    prm, hb = case(10, 9, 8, dict(DC.OPTIONS, equationType=eq))
    sums, h2 = oracle_free_stream_residual(DC.oracle_params(prm, 0.0, 0.0), hb)
    ref_totals(0.0, 0.0)
    r = rb.residual_core(_free_stream_prepared(prm, hb), prm, FLOW | TURB | INTERMED)
    ow = hb.d.owned()
    assert sums[1] > 0
    for l in range(hb.nw):
        _eq(r.a["dw"][ow + (l,)], h2.dw[ow + (l,)], "dw[%d]" % l)
