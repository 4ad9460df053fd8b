"""Multigrid on the device (adfb_mg_restrict, adfb_mg_prolong with both mgBoundCorr values, adfb_mg_cycle,
fullMultigridStartUp) on every boundary condition class, on split faces, on a polar axis and with the non-default
wall treatments, with the coarse levels built as the reference builds them (tests/mg_coarsen.py), against the oracle
compositions of test_mg_gpu.py / fmg_oracle.py -- which tests/test_oracle_vs_reference_mg_layouts.py pins bit for bit
against the reference on the same layouts.  Tolerances as test_mg_gpu.py / test_fmg_gpu.py hold the same entry points
to: 1e-13 on restricted states, 1e-12 / 1e-11 on residual-like arrays, 1e-9 on state changes."""
import numpy as np
import pytest

from adflow_b200.solver import ADFLOW_B200
from oracle.pyoracle import Oracle

import fmg_oracle as fo
import mg_coarsen as mc
from test_mg_gpu import device, oracle_mg_cycle, oracle_transfer_to_coarse, prepare_fine
from util import rel_l2, rel_max

pytestmark = pytest.mark.gpu

LIN = {"viscWallTreatment": "linear pressure extrapolation"}
EULER = {"equationType": "Euler"}
CASES = [("inout", (12, 9, 10), None, {}),
         ("inout", (13, 9, 11), EULER, {"outflowLinearExtrapol": 1, "reserved": 1}),
         ("supin", (11, 10, 9), LIN, {}),
         ("mixed", (12, 9, 10), dict(LIN, equationType="laminar NS"), {}),
         ("many", (11, 8, 9), EULER, {}),
         ("polar", (10, 12, 8), None, {})]
IDS = ["%s-%s" % (c[0], (c[2] or {}).get("equationType", "RANS").split()[0]) + ("-lin" if c[2] and "viscWallTreatment" in c[2] else "")
       for c in CASES]


def levels(c, nlev, **more):
    layout, shape, options, fields = c
    return mc.layout_levels(layout, shape, options, nlev, dict(fields, **more))


def c1(hb):
    d = hb.d
    return (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))


@pytest.mark.parametrize("neumann", [0, 1])
@pytest.mark.parametrize("c", CASES, ids=IDS)
def test_restrict_smooth_prolong(cuda_lib, c, neumann):
    prm, lv = levels(c, 2, mgBoundCorr=neumann)
    fine, coarse = lv
    s = device(prm, [hb.copy() for hb in lv])
    try:
        oracle_transfer_to_coarse(prm, fine, coarse)
        s.mgRestrict(1)
        ow, cc = coarse.d.owned(), c1(coarse)
        w, p, rlv, rev = s.downloadState(1)
        assert rel_max(w[cc][..., :5], coarse.w[cc][..., :5]) < 1e-13
        assert rel_max(p[cc], coarse.p[cc]) < 1e-13
        if prm.equations == 3:
            assert rel_max(rev[cc], coarse.rev[cc]) < 1e-13
        wr, dw, w1 = s.downloadArray(1, "wr", 5), s.downloadResidual(1), s.downloadArray(1, "w1", 5)
        for l in range(5):
            assert rel_l2(wr[ow + (l,)], coarse.wr[ow + (l,)]) < 1e-11, ("wr", l)
            assert rel_l2(dw[ow + (l,)], coarse.dw[ow + (l,)]) < 1e-12, ("dw", l)
        assert rel_max(w1[cc], coarse.w1[cc]) < 1e-13
        assert rel_max(s.downloadArray(1, "dtl")[ow], coarse.dtl[ow]) < 1e-12
        # the coarse-level BCs of every class inside the RK stages
        w0 = coarse.w.copy()
        Oracle(coarse, prm).rk_smoother()
        s.rkCycle(level=2)
        w, *_ = s.downloadState(1)
        for l in range(5):
            a, b = w[ow + (l,)] - w0[ow + (l,)], coarse.w[ow + (l,)] - w0[ow + (l,)]
            assert np.abs(b).max() > 0
            assert rel_l2(a, b) < 1e-9, ("coarse state change", l, rel_l2(a, b))
        # corrections with their boundary halos (setCorrectionsCoarseHalos), interpolation, fine BCs
        f0 = fine.w.copy()
        of, oc = Oracle(fine, prm), Oracle(coarse, prm)
        of.mg_prolong(oc)
        of.apply_flow_bc(True)
        s.mgProlong(1)
        wc, *_ = s.downloadState(1)
        assert rel_max(wc[cc][..., :5], coarse.w[cc][..., :5]) < 1e-9, ("coarse corrections", rel_max(wc[cc][..., :5], coarse.w[cc][..., :5]))
        w, p, rlv, rev = s.downloadState(0)
        owf = fine.d.owned()
        for l in range(5):
            a, b = w[owf + (l,)] - f0[owf + (l,)], fine.w[owf + (l,)] - f0[owf + (l,)]
            assert np.abs(b).max() > 0
            assert rel_l2(a, b) < 1e-9, ("fine correction", l, rel_l2(a, b))
        assert rel_max(w[..., :5], fine.w[..., :5]) < 1e-11
        assert rel_max(p, fine.p) < 1e-11
    finally:
        s.close()


CYCLE_CASES = [(CASES[0], "2v", 0), (CASES[0], "3w", 2), (CASES[1], "3w", 2), (CASES[2], "2v", 0),
               (CASES[2], "3w", 2), (CASES[4], "2v", 0)]


@pytest.mark.parametrize("c,cycle,dadi_sub", CYCLE_CASES,
                         ids=["%s-%s-%s" % (IDS[CASES.index(c)], cy, "DADI" if n else "RK") for c, cy, n in CYCLE_CASES])
def test_mg_cycle(cuda_lib, c, cycle, dadi_sub):
    """2V with the RK smoother and 3W with DADI over levels coarsened as the reference does"""
    prm, lv = levels(c, int(cycle[0]))
    dev = [hb.copy() for hb in lv]
    cyc = ADFLOW_B200.cycleStrategy(cycle)
    prepare_fine(Oracle(lv[0], prm))
    w0 = lv[0].w.copy()
    oracle_mg_cycle(prm, lv, cyc, dadi_subiter=dadi_sub)
    s = device(prm, dev)
    try:
        s.timeStep(False)
        s.smootherResidual(0)
        if dadi_sub:
            s.mgCycle(cyc, smoother="DADI", n_subiterations=dadi_sub)
        else:
            s.mgCycle(cyc)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    fine = lv[0]
    ow = fine.d.owned()
    for l in range(5):
        a, b = w[ow + (l,)] - w0[ow + (l,)], fine.w[ow + (l,)] - w0[ow + (l,)]
        assert np.abs(b).max() > 0
        assert rel_l2(a, b) < 1e-9, ("state change over the cycle", l, rel_l2(a, b))
    assert rel_max(w[..., :5], fine.w[..., :5]) < 1e-9


@pytest.mark.parametrize("smoother", ["RK", "DADI"])
@pytest.mark.parametrize("c", [CASES[0], CASES[3]], ids=[IDS[0], IDS[3]])
def test_full_multigrid_start_up_with_linear_wall_pressure(cuda_lib, c, smoother):
    """fullMultigridStartUp(3, ...) with linear pressure extrapolation at the walls: ground level 2 extrapolates
    linearly while level 3 above it takes constant pressure (adfb_set_ground_level's coarse flag)"""
    c = (c[0], c[1], dict(c[2] or {}, **LIN), c[3])
    prm, lv = levels(c, 3)
    assert not prm.wallBCConstantPressure
    oracle_transfer_to_coarse(prm, lv[0], lv[1])
    oracle_transfer_to_coarse(prm, lv[1], lv[2])
    for hb in lv:
        hb.fw[...] = 0
    dev = [hb.copy() for hb in lv]
    dadi = smoother == "DADI"
    snaps = fo.full_multigrid_start_up(prm, lv, 3, 2, "3w", dadi)
    s = device(prm, dev)
    got = {}
    try:
        prolong = s.mgProlongSolution

        def spy(fine_level=1):
            got[fine_level + 1] = s.downloadState(fine_level)[:2]
            prolong(fine_level)

        s.mgProlongSolution = spy
        s.fullMultigridStartUp(3, 2, "3w", smoother, 2)
        w, p = s.downloadState(0)[:2]
    finally:
        s.close()
    assert sorted(got) == sorted(snaps) == [2, 3]
    for ground in (3, 2):
        (wd, pd), (wo, po) = got[ground], snaps[ground]
        assert rel_max(wd, wo) < 1e-9, ("ground level %d" % ground, rel_max(wd, wo))
        assert rel_max(pd, po) < 1e-9
    assert rel_max(w, lv[0].w) < 1e-9, ("fine state after the start-up", rel_max(w, lv[0].w))
    assert rel_max(p, lv[0].p) < 1e-9
