"""Dissipation-based continuation and the free-stream residual on the device, against the oracle with the coefficients
of tests/diss_continuation.py (pinned to the reference's own routines in test_oracle_vs_reference_diss_continuation.py).

The states are flow regimes of tests/regimes.py in which the entropy / pressure sensor fires, so that the continuation
term is more than 1e3 x the tolerance of each row (checked on the CPU by that file).  Tolerances are those of the
entry points' parity tests: 1e-12 on residuals, 1e-10 / 1e-9 on state changes over a smoother cycle or step."""
import os

import numpy as np
import pytest

import diss_continuation as DC
import regimes as R
from adflow_b200.solver import ADFLOW_B200, RES_DISS_APPROX, RES_FLOW, RES_SKIP_PREAMBLE, RES_TURB, RES_UPDATE_INTERMED
from oracle.pyoracle import Oracle
from test_oracle_vs_reference_diss_continuation import oracle_free_stream_residual
from util import oracle_form_function, rel_l2, rel_max

pytestmark = pytest.mark.gpu

TOL = 1e-12
SHAPE = (12, 10, 8)
FT = RES_FLOW | RES_TURB


def _case(regime, eq="RANS", shape=SHAPE, **options):
    prm, hb = R.regime_case(regime, shape, dict(DC.OPTIONS, equationType=eq, **options))
    Oracle(hb, prm).reference_shock_sensor()
    return prm, hb


def _rows_close(got, want, hb, rows, tol, what="dw"):
    ow = hb.d.owned()
    for l in rows:
        a, b = got[ow + (l,)], want[ow + (l,)]
        assert np.isfinite(a).all(), (what, l)
        assert rel_l2(a, b) < tol, "%s[%d] rel L2 %.3e" % (what, l, rel_l2(a, b))


def _device_residual(prm, hbs, totals, flags, env=None):
    old = {k: os.environ.get(k) for k in (env or {})}
    os.environ.update(env or {})
    s = ADFLOW_B200(prm)
    try:
        for hb in hbs:
            s.addBlock(hb)
        s.setTotalResiduals(*totals)
        if flags & RES_DISS_APPROX:   # the approximate dissipation reads the frozen shock sensor
            s.referenceShockSensor()
        s.residual(flags)
        return [s.downloadResidual(b) for b in range(len(hbs))]
    finally:
        s.close()
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _oracle_core(prm, hb, flags, totals, rfil=1.0, approx=False):
    ho = hb.copy()
    Oracle(ho, DC.oracle_params(prm, *totals, approx=approx)).residual_core(flags, rfil)
    return ho


# ---------------------------------------------------------------------------------------------------------------------
# full residual: tile kernel (host-chosen tiles, ADFB_TILE seams) and the general kernels
@pytest.mark.parametrize("totals", DC.TOTALS)
@pytest.mark.parametrize("eq", ["RANS", "laminar NS", "Euler"])
@pytest.mark.parametrize("env", [{}, {"ADFB_TILE": "9,5,4"}, {"ADFB_FUSED": "0"}], ids=["tile", "seams", "general"])
def test_residual(cuda_lib, env, eq, totals):
    prm, hb = _case("supersonic", eq)
    flags = RES_FLOW | (RES_TURB if eq == "RANS" else 0)
    ref = _oracle_core(prm, hb, flags, totals)
    (dw,) = _device_residual(prm, [hb], totals, flags | RES_SKIP_PREAMBLE, env)
    _rows_close(dw, ref.dw, hb, range(hb.nw if eq == "RANS" else 5), TOL)


def test_residual_on_blocks_of_different_shapes(cuda_lib):
    totals = DC.TOTALS[1]
    cases = [_case(r, shape=sh) for r, sh in (("supersonic", (12, 10, 8)), ("contact_pocket", (9, 14, 6)),
                                               ("supersonic", (20, 7, 11)))]
    prm = cases[0][0]
    hbs = [hb for _, hb in cases]
    dws = _device_residual(prm, hbs, totals, FT | RES_SKIP_PREAMBLE)
    for hb, dw in zip(hbs, dws):
        _rows_close(dw, _oracle_core(prm, hb, FT, totals).dw, hb, range(6), TOL)


@pytest.mark.parametrize("totals", DC.TOTALS + [(0.0, 0.0)])
def test_approximate_residual(cuda_lib, totals):
    """the residual of the ANK operator (ADFB_RES_DISS_APPROX): the unguarded coefficient, NaN when both totals are 0"""
    prm, hb = _case("supersonic")
    ref = _oracle_core(prm, hb, FT | RES_DISS_APPROX, totals, approx=True)
    (dw,) = _device_residual(prm, [hb], totals, FT | RES_DISS_APPROX | RES_SKIP_PREAMBLE)
    ow = hb.d.owned()
    if totals == (0.0, 0.0):
        assert np.isnan(ref.dw[ow + (0,)]).all() and np.isnan(dw[ow + (0,)]).all()
        return
    _rows_close(dw, ref.dw, hb, range(6), TOL)


@pytest.mark.parametrize("disc", ["central plus matrix dissipation", "upwind"])
def test_no_effect_without_scalar_dissipation(cuda_lib, disc):
    prm, hb = _case("supersonic", discretization=disc)
    (on,) = _device_residual(prm, [hb], DC.TOTALS[1], FT | RES_SKIP_PREAMBLE)
    (off,) = _device_residual(DC.plain(prm), [hb], DC.TOTALS[1], FT | RES_SKIP_PREAMBLE)
    assert np.array_equal(on, off)


# ---------------------------------------------------------------------------------------------------------------------
# smoothers
def _smoother_start(prm, hb, totals):
    ho = hb.copy()
    o = Oracle(ho, DC.oracle_params(prm, *totals))
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(prm.cdisRK[0])
    return ho, o


def _device_smoother(prm, hb, totals, step):
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.setTotalResiduals(*totals)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        dw0 = s.downloadResidual(0)
        step(s)
        return dw0, s.downloadState(0), s.downloadResidual(0)
    finally:
        s.close()


@pytest.mark.parametrize("totals", DC.TOTALS[:4])
def test_smoother_residual_and_rk_cycle(cuda_lib, totals):
    prm, hb = _case("contact_pocket", nRKStages=5, resAveraging="never")
    ho, o = _smoother_start(prm, hb, totals)
    dw0 = ho.dw.copy()
    o.rk_smoother()
    dw_dev0, (w, p, rlv, rev), _ = _device_smoother(prm, hb, totals, lambda s: s.rkCycle())
    _rows_close(dw_dev0, dw0, hb, range(5), TOL, "smoother dw")
    ow = hb.d.owned()
    for l in range(5):
        dv, do = w[ow + (l,)] - hb.w[ow + (l,)], ho.w[ow + (l,)] - hb.w[ow + (l,)]
        assert rel_l2(dv, do) < 1e-10, ("state change", l, rel_l2(dv, do))


@pytest.mark.parametrize("totals", [DC.TOTALS[1], DC.TOTALS[4]])
def test_dadi_step_and_sa_ddadi(cuda_lib, totals):
    prm, hb = _case("contact_pocket")
    ho, o = _smoother_start(prm, hb, totals)
    o.dadi_step()
    o.sa_block()
    _, (w, p, rlv, rev), dw = _device_smoother(prm, hb, totals, lambda s: (s.dadiStep(), s.turbSolveDDADI(1)))
    ow = hb.d.owned()
    for l in range(6):
        dv, do = w[ow + (l,)] - hb.w[ow + (l,)], ho.w[ow + (l,)] - hb.w[ow + (l,)]
        assert rel_l2(dv, do) < 1e-9, ("state change", l, rel_l2(dv, do))


# ---------------------------------------------------------------------------------------------------------------------
# Newton-Krylov: form function (one-shot and pipelined) and the matrix-free product
@pytest.mark.parametrize("pipe", ["1", "6"])
def test_form_function_and_mffd(cuda_lib, pipe):
    totals = DC.TOTALS[1]
    prm, hb = _case("supersonic", shape=(12, 10, 16))
    U = np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()
    a = np.random.default_rng(5).standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-7
    po = DC.oracle_params(prm, *totals)
    ref, ref1 = oracle_form_function(po, hb, U), oracle_form_function(po, hb, U + h * a)
    old = os.environ.get("ADFB_FF_PIPE")
    os.environ["ADFB_FF_PIPE"] = pipe
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.setTotalResiduals(*totals)
        r = s.formFunction(U)
        s.mffdSetBase(U)
        y = s.mffdApply(a, h)
    finally:
        s.close()
        if old is None:
            os.environ.pop("ADFB_FF_PIPE", None)
        else:
            os.environ["ADFB_FF_PIPE"] = old
    assert rel_l2(r, ref) < TOL, rel_l2(r, ref)
    assert rel_l2(r, oracle_form_function(DC.plain(prm), hb, U)) > 1e3 * TOL
    assert rel_l2(y, (ref1 - ref) / h) < 1e-4


# ---------------------------------------------------------------------------------------------------------------------
# graphs: new totals between replays re-use the recorded graphs and give the bits of a fresh context
def test_totals_between_graph_replays(cuda_lib):
    prm, hb = _case("supersonic")
    seq = [DC.TOTALS[0], DC.TOTALS[1], DC.TOTALS[3], DC.TOTALS[1]]
    fresh = {t: _device_residual(prm, [hb], t, FT)[0] for t in set(seq)}
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        counts = []
        for t in seq:
            s.setTotalResiduals(*t)
            s.residual(FT)
            assert np.array_equal(s.downloadResidual(0), fresh[t]), t
            s.uploadState(0, hb)
            counts.append(s.graphCount())
    finally:
        s.close()
    assert counts[0] >= 1 and len(set(counts)) == 1, counts
    assert not np.array_equal(fresh[DC.TOTALS[0]], fresh[DC.TOTALS[1]])


# ---------------------------------------------------------------------------------------------------------------------
# a short host-driven run: totalR0 from the device free-stream residual, totalR from each cycle's residual
def test_host_driven_runge_kutta_run(cuda_lib):
    prm, hb = _case("contact_pocket", "Euler", shape=(16, 12, 10), resAveraging="never")
    s = ADFLOW_B200(prm)
    dev = []
    try:
        s.addBlock(hb)
        tr0 = s.getFreeStreamResidual()
        tr = 0.0
        s.applyBCs(True, True)
        for _ in range(10):
            s.setTotalResiduals(tr, tr0)
            s.timeStep(False)
            s.smootherResidual(0)
            tr = float(np.sqrt(s.getResNorms()[1]))
            dev.append(tr)
            s.rkCycle()
    finally:
        s.close()
    ref = []
    ho = hb.copy()
    otr0 = float(np.sqrt(oracle_free_stream_residual(prm, hb)[0][1]))
    assert abs(otr0 - tr0) <= 1e-10 * otr0
    otr = 0.0
    Oracle(ho, DC.plain(prm)).apply_flow_bc(True)
    for _ in range(10):
        o = Oracle(ho, DC.oracle_params(prm, otr, otr0))
        o.time_step(True)
        ho.fw[...] = 0
        o.residual_block(prm.cdisRK[0])
        otr = float(np.sqrt(o.norms()[1]))
        ref.append(otr)
        o.rk_smoother()
    dev, ref = np.array(dev), np.array(ref)
    assert np.abs(dev - ref).max() <= 1e-7 * ref.max(), (dev, ref)
    assert ref[-1] != ref[0]


# ---------------------------------------------------------------------------------------------------------------------
# free-stream residual
@pytest.mark.parametrize("eq,continuation", [("RANS", True), ("RANS", False), ("laminar NS", True), ("Euler", True)])
def test_free_stream_residual(cuda_lib, eq, continuation):
    """the sums against the oracle; afterwards the block holds exactly what a plain adfb_residual(FLOW | TURB |
    UPDATE_INTERMED) of the uploaded state leaves: w, p, rlv, rev with halos, dw, dtl and the radii (a second context)"""
    import ctypes as C

    prm, hb = _case("supersonic", eq)
    if not continuation:
        prm = DC.plain(prm)
    want, _ = oracle_free_stream_residual(DC.oracle_params(prm, 0.0, 0.0), hb)
    out = (C.c_double * 2)()
    got = {}
    for name in ("free stream", "plain"):
        s = ADFLOW_B200(prm)
        try:
            s.addBlock(hb)
            if name == "plain":
                s.residual(FT | RES_UPDATE_INTERMED)
            else:
                assert s.L.adfb_free_stream_residual(out) == 0
            got[name] = list(s.downloadState(0)) + [s.downloadResidual(0)] + list(s.downloadIntermed(0).values())
            if name != "plain":
                total = s.getFreeStreamResidual()
        finally:
            s.close()
    sums = np.array([out[0], out[1]])
    assert want[1] > 0
    assert np.all(np.abs(sums - want) <= 1e-10 * want), (sums, want)
    assert total == np.sqrt(out[1])
    for q, (a, b) in enumerate(zip(got["free stream"], got["plain"])):
        assert np.array_equal(a, b), q


def test_free_stream_residual_of_several_blocks(cuda_lib):
    import ctypes as C

    cases = [_case("supersonic", shape=sh) for sh in ((12, 10, 8), (9, 14, 6), (7, 8, 11))]
    prm = cases[0][0]
    want = sum(oracle_free_stream_residual(DC.oracle_params(prm, 0.0, 0.0), hb)[0] for _, hb in cases)
    s = ADFLOW_B200(prm)
    try:
        for _, hb in cases:
            s.addBlock(hb)
        out = (C.c_double * 2)()
        assert s.L.adfb_free_stream_residual(out) == 0
    finally:
        s.close()
    got = np.array([out[0], out[1]])
    assert np.all(np.abs(got - want) <= 1e-10 * want), (got, want)
