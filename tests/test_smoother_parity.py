"""Parity of the device BC / Runge-Kutta / residual-averaging kernels with the oracle."""
import numpy as np
import pytest

from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
from oracle.pyoracle import Oracle

from util import case, rel_l2, rel_max

pytestmark = pytest.mark.gpu


def box_close(a, b, tol, name):
    assert np.isfinite(a).all(), name
    err = rel_max(a, b)
    assert err < tol, "%s: rel max %.3e" % (name, err)


ISO_EXTRAP_FACES = {1: 5, 2: 3, 3: 1, 4: 3, 5: 6, 6: 5}  # iMin extrap, jMin symm, kMin isothermal wall, kMax extrap
INOUT_FACES = {1: 8, 2: 7, 3: 9, 4: 10, 5: 2, 6: 8}      # subsonic in (total) / out, supersonic in / out, wall, subsonic in (mass flow)
POLAR_FACES = {1: 11, 2: 3, 3: 1, 4: 11, 5: 2, 6: 11}    # polar symmetry on a min and two max faces


@pytest.mark.parametrize("options,faces", [(None, None), ({"equationType": "Euler"}, None),
                                           ({"equationType": "laminar NS"}, None),
                                           ({"viscWallTreatment": "linear pressure extrapolation"}, None),
                                           (None, ISO_EXTRAP_FACES),
                                           ({"viscWallTreatment": "linear pressure extrapolation"}, ISO_EXTRAP_FACES),
                                           (None, INOUT_FACES), ({"equationType": "Euler"}, INOUT_FACES),
                                           (None, POLAR_FACES)])
def test_bcs_match_oracle(cuda_lib, options, faces):
    prm, hb = case(13, 11, 9, options, **({} if faces is None else {"physical_faces": faces}))
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True)
    o.apply_flow_bc(True)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    assert np.abs(w - hb.w).max() > 0  # the BCs changed the halos
    box_close(w, ho.w, 1e-13, "w")
    box_close(p, ho.p, 1e-13, "p")
    box_close(rlv, ho.rlv, 1e-13, "rlv")
    box_close(rev, ho.rev, 1e-13, "rev")


def test_full_residual_with_preamble(cuda_lib):
    """adfb_residual without SKIP_PREAMBLE == blocketteRes :199-283 on one block."""
    prm, hb = case(14, 10, 9)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.residual_core(RES_FLOW | RES_TURB)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.residual(RES_FLOW | RES_TURB)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(6):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-12, l


@pytest.mark.parametrize("options", [
    {"nRKStages": 5, "resAveraging": "alternate"},
    {"nRKStages": 5, "resAveraging": "never"},
    {"equationType": "Euler", "nRKStages": 3, "resAveraging": "never"},
    {"equationType": "Euler", "nRKStages": 4, "resAveraging": "always", "CFL": 4.0},
    {"discretization": "central plus matrix dissipation", "nRKStages": 5, "resAveraging": "never"},
    {"discretization": "upwind", "equationType": "Euler", "nRKStages": 3, "resAveraging": "never"},
    {"discretization": "central plus matrix dissipation", "equationType": "Euler", "nRKStages": 3, "resAveraging": "never"},
    {"discretization": "upwind", "equationType": "laminar NS", "nRKStages": 5, "resAveraging": "never"},
    {"discretization": "upwind", "nRKStages": 5, "resAveraging": "never"},
])
def test_rk_cycle_matches_oracle(cuda_lib, options):
    prm, hb = case(16, 12, 10, options)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(prm.cdisRK[0])
    dw0 = ho.dw.copy()
    o.rk_smoother()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        dw_dev0 = s.downloadResidual(0)
        s.rkCycle()
        w, p, rlv, rev = s.downloadState(0)
        dw_dev = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw_dev0[ow + (l,)], dw0[ow + (l,)]) < 1e-12, ("dw before cycle", l)
    # the state after nRKStages updates; the change over a cycle is what is compared tightly
    dwv = w[ow] - hb.w[ow]
    dwo = ho.w[ow] - hb.w[ow]
    assert np.abs(dwo[..., :5]).max() > 1e-8
    for l in range(5):
        assert rel_l2(dwv[..., l], dwo[..., l]) < 1e-10, ("state change", l, rel_l2(dwv[..., l], dwo[..., l]))
    box_close(w[..., :5], ho.w[..., :5], 1e-11, "w after RK cycle (halos included)")
    box_close(p, ho.p, 1e-11, "p after RK cycle")
    if prm.equations != 1:
        d = hb.d
        c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
        box_close(rlv[c1], ho.rlv[c1], 1e-11, "rlv")


@pytest.mark.parametrize("shape", [(18, 7, 9), (20, 17, 16), (36, 19, 41)])
def test_residual_averaging_matches_oracle(cuda_lib, shape):
    prm, hb = case(*shape, {"CFL": 6.0, "resAveraging": "always", "nRKStages": 1})
    # one RK stage with averaging: compare dw after the stage (scaled + smoothed)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(1.0)
    np.copyto(ho.wn, ho.w[..., :5]); np.copyto(ho.pn, ho.p)
    o.rk_stage(1)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.timeStep(False)
        s.smootherResidual(0)
        s.rkCycle()
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-11, l
