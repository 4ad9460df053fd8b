"""The multigrid pins of test_oracle_vs_reference_mg.py / test_oracle_vs_reference_fmg.py on every boundary condition
class, on faces split into pieces, on a polar axis and with the non-default wall and correction treatments, with the
coarse levels built as the reference builds them (tests/mg_coarsen.py): the oracle BIT FOR BIT against the reference's
own transferToCoarseGrid, transferToFineGrid, RungeKuttaSmoother, DADISmoother and executeMGCycle (translated,
oracle/_ref).  Skipped where the translated library is absent."""
import numpy as np
import pytest

from oracle import refblockette as rb
from oracle.pyoracle import Oracle

import mg_coarsen as mc
from test_oracle_vs_reference_mg import eq, oracle_transfer_to_coarse

pytestmark = pytest.mark.skipif(not rb.available(), reason="oracle/_ref not built (no /root/reference at build time)")

LIN = {"viscWallTreatment": "linear pressure extrapolation"}
EULER = {"equationType": "Euler"}
# (layout, shape, options, parameter fields); odd and even cell counts, so that irregular coarse cells sit at max ends,
# inside lines next to subface ends and, on level 3, at min ends
MATRIX = [
    ("inout", (12, 9, 10), None, {}),
    ("inout", (13, 9, 11), EULER, {"outflowLinearExtrapol": 1}),
    ("inout", (13, 9, 11), LIN, {"outflowLinearExtrapol": 1}),
    ("inout", (12, 9, 10), EULER, {"reserved": 1}),
    ("supin", (11, 10, 9), None, {}),
    ("supin", (11, 10, 9), dict(EULER, resAveraging="never"), {"reserved": 1}),
    ("mixed", (12, 9, 10), None, {}),
    ("mixed", (12, 9, 10), dict(LIN, equationType="laminar NS"), {}),
    ("many", (11, 8, 9), EULER, {}),
    ("polar", (10, 12, 8), None, {}),
    ("polar", (10, 12, 8), dict(LIN, equationType="laminar NS"), {}),
]


def _id(m):
    layout, shape, options, fields = m
    opts = ",".join("%s=%s" % (k, str(v).split()[0]) for k, v in sorted((options or {}).items()))
    flds = ",".join("%s=%s" % kv for kv in sorted(fields.items()))
    return "-".join(x for x in (layout, "x".join(map(str, shape)), opts, flds) if x)


IDS = [_id(m) for m in MATRIX]


def levels(m, nlev=2, **more):
    layout, shape, options, fields = m
    return mc.layout_levels(layout, shape, options, nlev, dict(fields, **more))


def c1(hb):
    d = hb.d
    return (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))


@pytest.mark.parametrize("m", MATRIX, ids=IDS)
def test_transfer_to_coarse_grid(m):
    prm, (fine, coarse) = levels(m)
    f2, c2 = fine.copy(), coarse.copy()
    mg = rb.RefMG(f2, c2, prm)
    try:
        mg.transfer_to_coarse()
    finally:
        mg.close()
    rf, rc = mg.lv[1].a, mg.lv[2].a
    oracle_transfer_to_coarse(prm, fine, coarse)
    ow, cc = coarse.d.owned(), c1(coarse)
    eq(coarse.wr[ow], rc["wr"][ow], "wr (forcing term)")
    eq(coarse.dw[ow][..., :5], rf["dw"][ow][..., :5], "coarse dw")
    eq(coarse.w[cc][..., :5], rc["w"][cc][..., :5], "coarse w incl. first halos")
    eq(coarse.p[cc], rc["p"][cc], "coarse p")
    eq(coarse.w1[cc], rc["w1"][cc], "w1")
    eq(coarse.dtl[ow], rf["dtl"][ow], "coarse dtl")
    if prm.equations == 3:
        eq(coarse.rev[cc], rc["rev"][cc], "coarse rev")


@pytest.mark.parametrize("smoother", ["RK", "DADI"])
@pytest.mark.parametrize("m", MATRIX, ids=IDS)
def test_coarse_level_smoother(m, smoother):
    """RungeKuttaSmoother / DADISmoother (one step) on level 2: the coarse-level BCs of every class, first halos only"""
    prm, (fine, coarse) = levels(m)
    oracle_transfer_to_coarse(prm, fine, coarse)
    f2, c2 = fine.copy(), coarse.copy()
    mg = rb.RefMG(f2, c2, prm)
    try:
        mg.seed_coarse_shared()
        if smoother == "RK":
            mg.call(2, "smoothers_rungekuttasmoother")
        else:
            rb.set_int("smoother", 2); rb.set_int("nsubiterations", 1); rb.set_int("rkstage", 0)
            mg.call(2, "smoothers_dadismoother")
    finally:
        rb.set_int("smoother", 1); rb.set_int("nsubiterations", 1)
        mg.close()
    rc = mg.lv[2].a
    oc = Oracle(coarse, prm)
    oc.rk_smoother() if smoother == "RK" else oc.dadi_step()
    d, cc = coarse.d, c1(coarse)
    assert np.abs(coarse.w[d.owned()][..., :5] - c2.w[d.owned()][..., :5]).max() > 0
    eq(coarse.w[cc][..., :5], rc["w"][cc][..., :5], "coarse w after the smoother")
    eq(coarse.p[cc], rc["p"][cc], "coarse p after the smoother")


@pytest.mark.parametrize("neumann", [0, 1])
@pytest.mark.parametrize("m", MATRIX, ids=IDS)
def test_transfer_to_fine_grid(m, neumann):
    """transferToFineGrid(.true.) with mgBoundCorr = bcDirichlet0 / bcNeumann: setCorrectionsCoarseHalos on every
    subface in BCData order, the interpolation (irregular cells included), the fine BCs"""
    prm, (fine, coarse) = levels(m, mgBoundCorr=neumann)
    oracle_transfer_to_coarse(prm, fine, coarse)
    Oracle(coarse, prm).rk_smoother()
    f2, c2 = fine.copy(), coarse.copy()
    mg = rb.RefMG(f2, c2, prm)
    try:
        mg.transfer_to_fine()
    finally:
        mg.close()
    rf, rc = mg.lv[1].a, mg.lv[2].a
    of, oc = Oracle(fine, prm), Oracle(coarse, prm)
    of.mg_prolong(oc)
    of.apply_flow_bc(True)
    cc, ow = c1(coarse), fine.d.owned()
    eq(coarse.w[cc][..., :5], rc["w"][cc][..., :5], "corrections on the coarse block (incl. boundary halos)")
    eq(fine.dw[ow][..., :5], rf["dw"][ow][..., :5], "interpolated corrections")
    assert np.abs(fine.w[ow][..., :5] - f2.w[ow][..., :5]).max() > 0
    eq(fine.w[..., :5], rf["w"][..., :5], "fine w (whole box)")
    eq(fine.p, rf["p"], "fine p")
    if prm.equations == 3:
        eq(fine.rev, rf["rev"], "fine rev")


@pytest.mark.parametrize("m", MATRIX, ids=IDS)
def test_full_multigrid_start_up_transfer(m):
    """transferToFineGrid(.false.): the coarse solution with its corrected halos (fact 1) interpolated, halos
    extrapolated, turbulence and flow BCs with second halos"""
    prm, (fine, coarse) = levels(m)
    oracle_transfer_to_coarse(prm, fine, coarse)
    Oracle(coarse, prm).rk_smoother()
    rng = np.random.default_rng(5)
    fine.w[...] = fine.w * (1.0 + 0.05 * rng.standard_normal(fine.w.shape))
    f2, c2 = fine.copy(), coarse.copy()
    mg = rb.RefMG(f2, c2, prm)
    try:
        mg.transfer_to_fine(corrections=False)
    finally:
        mg.close()
    rf, rc = mg.lv[1].a, mg.lv[2].a
    of, oc = Oracle(fine, prm), Oracle(coarse, prm)
    of.mg_prolong_solution(oc)
    if prm.equations == 3:
        of.apply_turb_bc(True)
    of.apply_flow_bc(True); of.apply_flow_bc(True); of.apply_flow_bc(True)
    cc = c1(coarse)
    eq(coarse.w[cc], rc["w"][cc], "coarse w with the pressure in place of rho*E (incl. boundary halos)")
    eq(fine.w, rf["w"], "fine w (whole box)")
    eq(fine.p, rf["p"], "fine p")
    if prm.equations == 3:
        eq(fine.rev, rf["rev"], "fine rev")


@pytest.mark.parametrize("m", MATRIX, ids=IDS)
def test_rk_smoother_on_a_coarse_ground_level(m):
    """RungeKuttaSmoother with currentLevel = groundLevel = 2: the fine-grid routines and BCs on the coarse block --
    so the wall BCs take the treatment the parameters ask for instead of constant pressure"""
    prm, (fine, coarse) = levels(m)
    oracle_transfer_to_coarse(prm, fine, coarse)
    cfl = prm.cfl
    try:
        prm.cfl = prm.cflCoarse
        coarse.level = 1
        og = Oracle(coarse, prm)
        if prm.equations == 3:
            og.apply_turb_bc(True)
        og.apply_flow_bc(True)
        og.time_step(True)
        coarse.fw[...] = 0
        og.residual_block(prm.cdisRK[0])
        f2, c2 = fine.copy(), coarse.copy()
        c2.level = 2
        prm.cfl = cfl
        mg = rb.RefMG(f2, c2, prm)
        try:
            mg.seed_coarse_shared()
            mg.call(2, "smoothers_rungekuttasmoother", ground=2)
        finally:
            mg.close()
        rc = mg.lv[2].a
        prm.cfl = prm.cflCoarse
        og.rk_smoother()
    finally:
        prm.cfl = cfl
        coarse.level = 2
    eq(coarse.w[..., :5], rc["w"][..., :5], "coarse-ground-level w after the RK cycle (whole box, second halos)")
    eq(coarse.p, rc["p"], "p")
    if prm.equations == 3:
        eq(coarse.rev, rc["rev"], "rev")


# No polar block here: its j faces are a periodic cut that no BC writes, and without the cut's exchange the
# reference's coarse rlv halos there are whatever the finest level left in the array every level shares (setPointers);
# the oracle's levels own their arrays.  The single transfers and smoothers above do not read those halos.
CYCLES = [(MATRIX[0], "3w", 0), (MATRIX[2], "3v", 0), (MATRIX[3], "2v", 0), (MATRIX[5], "3w", 2), (MATRIX[6], "3w", 0),
          (MATRIX[8], "2v", 0)]


@pytest.mark.parametrize("m,cycle,dadi_sub", CYCLES, ids=["%s-%s-%s" % (_id(m), c, "DADI" if s else "RK") for m, c, s in CYCLES])
def test_execute_mg_cycle_driven_by_the_reference(m, cycle, dadi_sub):
    """executeMGCycle of the reference over levels coarsened as the reference coarsens them, against the composition
    of the oracle's pieces the device is held to (test_mg_gpu.oracle_mg_cycle)"""
    from adflow_b200.solver import ADFLOW_B200
    from test_mg_gpu import oracle_mg_cycle, prepare_fine

    prm, lv = levels(m, int(cycle[0]))
    prepare_fine(Oracle(lv[0], prm))
    cyc = ADFLOW_B200.cycleStrategy(cycle)
    ref = [hb.copy() for hb in lv]
    mg = rb.RefMG(ref[0], ref[1], prm, more_levels=ref[2:])
    try:
        mg.execute_mg_cycle(cyc, smoother="DADI" if dadi_sub else "RK", n_subiterations=max(dadi_sub, 1))
    finally:
        mg.close()
    rf = mg.lv[1].a
    fine = lv[0]
    w0 = fine.w.copy()
    oracle_mg_cycle(prm, lv, cyc, dadi_subiter=dadi_sub)
    ow = fine.d.owned()
    assert np.abs(fine.w[ow] - w0[ow]).max() > 0
    eq(fine.w[..., :fine.nw], rf["w"][..., :fine.nw], "fine state after the cycle (whole box)")
    eq(fine.p, rf["p"], "fine p")
    eq(fine.dw[ow][..., :5], rf["dw"][ow][..., :5], "fine residual after the cycle")
