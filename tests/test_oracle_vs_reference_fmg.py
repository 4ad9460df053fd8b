"""Pin the oracle on a coarse GROUND level (the full-multigrid start-up, src/solver/solvers.F90:63-117) with a coarse
discretisation other than the fine one, BIT FOR BIT against the reference's own routines (translated, oracle/_ref):

* solveState's start on ground level 2 (solvers.F90:1014-1018): blocketteResCore selects spaceDiscr on every level
  (blockette.F90:637-653), then timeStep(.false.);
* RungeKuttaSmoother / DADISmoother from that residual: every later residual is residual_block with discr =
  spaceDiscrCoarse (currentLevel /= 1) and fineGrid = .true. (residuals.F90:71-75), i.e. the fine-grid routine of the
  coarse discretisation;
* transferToCoarseGrid from ground level 2 to level 3: its timeStep(.true.) returns at once unless the fine discretisation
  is scalar dissipation (radiiNeededFine, solverUtils.F90:90-96), so the residual reads the radii of the last
  timeStep(.false.) -- unscaled unless spaceDiscr is scalar dissipation (dirScaling, inputParamRoutines.F90:2824);
* one whole executeMGCycle (2V) on ground level 2 over levels 2-3 (multiGrid.F90:825-955).

Skipped where the translated library is absent."""
import numpy as np
import pytest

from adflow_b200 import synthetic as syn
from adflow_b200.solver import ADFLOW_B200
from oracle import refblockette as rb
from oracle.pyoracle import Oracle

import fmg_oracle as fo
from util import case

pytestmark = pytest.mark.skipif(not rb.available(), reason="oracle/_ref not built (no /root/reference at build time)")

SC, MA, UP = "central plus scalar dissipation", "central plus matrix dissipation", "upwind"
# every off-diagonal (discretization, coarseDiscretization) pair with Euler; the pyADflow default coarse discretisation
# (scalar) under matrix and upwind fine discretisations with laminar NS and RANS-SA
PAIRS = ([("Euler", f, c) for f in (SC, MA, UP) for c in (SC, MA, UP) if f != c]
         + [(eq, f, SC) for eq in ("laminar NS", "RANS") for f in (MA, UP)])
IDS = ["%s-%s-%s" % (eq.split()[0], f.split()[-2] if f != UP else "upwind", c.split()[-2] if c != UP else "upwind")
       for eq, f, c in PAIRS]


def eq_(a, b, name):
    assert np.isfinite(a).all(), name
    assert np.array_equal(a, b), "%s: max |diff| %.3e" % (name, np.abs(a - b).max())


def three_levels(eqn, fine_disc, coarse_disc, shape=(16, 12, 8)):
    """levels 1, 2, 3 of one block; level 2 carries the restriction of the fine state (ground-level-1 transfer) and is
    then prepared as ground level 2 like blocketteRes' preamble: p, rlv, rev, BCs."""
    prm, fine = case(*shape, {"equationType": eqn, "discretization": fine_disc, "coarseDiscretization": coarse_disc})
    fine.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    o = Oracle(fine, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    l2 = syn.make_coarse_block(fine, prm)
    l3 = syn.make_coarse_block(l2, prm)
    of, oc = Oracle(fine, prm), Oracle(l2, prm)
    of.time_step(False); of.residual_block(prm.cdisRK[0])
    oc.mg_restrict(of); oc.apply_flow_bc(False)
    for hb in (fine, l2, l3):
        hb.fw[...] = 0
    fo.Ground(l2, prm).preamble()
    return prm, [fine, l2, l3]


def ref_start(mg):
    """the same with the reference's blocketteResCore and timeStep_block on level 2"""
    flags = (0, 0, 0, 1, 1, 0)   # approximate dissipation, approximate viscous flux, updateIntermed, flow, turbulence, storeWall
    mg.call(2, "blocketterescore", *flags, ground=2)
    mg.call(2, "solverutils_timestep_block", 0, ground=2)


def ref_levels(levels, prm):
    rl = [hb.copy() for hb in levels]
    mg = rb.RefMG(rl[0], rl[1], prm, more_levels=rl[2:])
    mg.seed_coarse_shared()
    return mg


def c1(d):
    return (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))


@pytest.mark.parametrize("eqn,fdisc,cdisc", PAIRS, ids=IDS)
def test_blockette_residual_on_a_coarse_ground_level(eqn, fdisc, cdisc):
    """rule of blocketteRes: spaceDiscr on every level, directional scaling always, whatever the coarse discretisation"""
    prm, levels = three_levels(eqn, fdisc, cdisc)
    l2 = levels[1]
    mg = ref_levels(levels, prm)
    try:
        mg.call(2, "blocketterescore", 0, 0, 1, 1, 1, 0, ground=2)
    finally:
        mg.close()
    rf = mg.lv[1].a
    fo.Ground(l2, prm).blockette_residual()
    ow = l2.d.owned()
    nv = l2.nw if prm.equations == 3 else 5
    eq_(l2.dw[ow][..., :nv], rf["dw"][ow][..., :nv], "blockette dw on ground level 2")
    eq_(l2.dtl[ow], rf["dtl"][ow], "dtl")
    for n, m in (("radI", "radi"), ("radJ", "radj"), ("radK", "radk")):
        eq_(getattr(l2, n)[c1(l2.d)], rf[m][c1(l2.d)], n)


def _smoother(eqn, fdisc, cdisc, dadi):
    prm, levels = three_levels(eqn, fdisc, cdisc)
    l2 = levels[1]
    mg = ref_levels(levels, prm)
    try:
        ref_start(mg)
        if dadi:   # DADISmoother: one step on a coarse ground level whatever nSubiterations says (smoothers.F90:400)
            rb.set_int("smoother", 2); rb.set_int("nsubiterations", 3); rb.set_int("rkstage", 0)
            mg.call(2, "smoothers_dadismoother", ground=2)
        else:
            mg.call(2, "smoothers_rungekuttasmoother", ground=2)
    finally:
        rb.set_int("smoother", 1); rb.set_int("nsubiterations", 1)
        mg.close()
    rc, rf = mg.lv[2].a, mg.lv[1].a
    w0 = l2.w.copy()
    g = fo.Ground(l2, prm)
    g.start()
    if dadi:
        g.block().dadi_step()
    else:
        g.block().rk_smoother()
    d = l2.d
    assert np.abs(l2.w[d.owned()][..., :5] - w0[d.owned()][..., :5]).max() > 0
    eq_(l2.w[..., :5], rc["w"][..., :5], "ground-level-2 w after the smoother (whole box, second halos)")
    eq_(l2.p, rc["p"], "p")
    eq_(l2.dw[d.owned()][..., :5], rf["dw"][d.owned()][..., :5], "dw")
    if prm.equations == 3:
        eq_(l2.rev, rc["rev"], "rev")


@pytest.mark.parametrize("eqn,fdisc,cdisc", PAIRS, ids=IDS)
def test_rk_smoother_from_the_blockette_residual(eqn, fdisc, cdisc):
    _smoother(eqn, fdisc, cdisc, dadi=False)


@pytest.mark.parametrize("eqn,fdisc,cdisc", PAIRS, ids=IDS)
def test_dadi_smoother_from_the_blockette_residual(eqn, fdisc, cdisc):
    _smoother(eqn, fdisc, cdisc, dadi=True)


@pytest.mark.parametrize("eqn,fdisc,cdisc", PAIRS, ids=IDS)
def test_transfer_to_coarse_grid_from_ground_level_2(eqn, fdisc, cdisc):
    """after an RK cycle, so that the radii of the last timeStep(.false.) belong to an older state than the residual's:
    with fine = matrix or upwind and coarse = scalar the scalar dissipation of the level-2 residual reads those"""
    prm, levels = three_levels(eqn, fdisc, cdisc)
    l2, l3 = levels[1], levels[2]
    mg = ref_levels(levels, prm)
    try:
        ref_start(mg)
        mg.call(2, "smoothers_rungekuttasmoother", ground=2)
        rb.set_int("currentlevel", 2); rb.set_int("groundlevel", 2); rb.set_int("rkstage", 0)
        rb.lib().multigrid_transfertocoarsegrid()
    finally:
        rb.set_int("groundlevel", 1)
        mg.close()
    rc, rf = mg.lv[3].a, mg.lv[1].a
    g = fo.Ground(l2, prm)
    g.start()
    g.block().rk_smoother()
    fo.transfer_to_coarse(prm, g, l3)
    d = l3.d
    ow = d.owned()
    eq_(l3.wr[ow], rc["wr"][ow], "wr (forcing term of level 3)")
    eq_(l3.w[c1(d)][..., :5], rc["w"][c1(d)][..., :5], "level-3 w incl. first halos")
    eq_(l3.p[c1(d)], rc["p"][c1(d)], "level-3 p")
    eq_(l3.dw[ow][..., :5], rf["dw"][ow][..., :5], "level-3 dw")
    eq_(l3.dtl[ow], rf["dtl"][ow], "level-3 dtl")


@pytest.mark.parametrize("eqn,fdisc,cdisc", PAIRS, ids=IDS)
def test_execute_mg_cycle_on_ground_level_2(eqn, fdisc, cdisc):
    """the reference's executeMGCycle (2V over levels 2-3, RK) on ground level 2 after solveState's start, against
    the oracle composition tests/test_fmg_gpu.py holds the device to"""
    prm, levels = three_levels(eqn, fdisc, cdisc)
    l2 = levels[1]
    cyc = ADFLOW_B200.cycleStrategy("2v")
    mg = ref_levels(levels, prm)
    try:
        ref_start(mg)
        arr = rb.C.c_int * 256
        cycling = arr.in_dll(rb.lib(), "cycling")
        for q, v in enumerate(cyc):
            cycling[q] = v
        rb.set_int("nstepscycling", len(cyc)); rb.set_int("rkstage", 0)
        rb.set_int("groundlevel", 2); rb.set_int("currentlevel", 2)
        rb.lib().multigrid_executemgcycle()
    finally:
        rb.set_int("groundlevel", 1)
        mg.close()
    rc, rf = mg.lv[2].a, mg.lv[1].a
    w0 = l2.w.copy()
    fo.Ground(l2, prm).start()
    fo.mg_cycle(prm, levels[1:], cyc)
    d = l2.d
    ow = d.owned()
    assert np.abs(l2.w[ow] - w0[ow]).max() > 0
    nv = l2.nw
    eq_(l2.w[..., :nv], rc["w"][..., :nv], "ground-level-2 state after the cycle (whole box)")
    eq_(l2.p, rc["p"], "p")
    eq_(l2.dw[ow][..., :5], rf["dw"][ow][..., :5], "residual after the cycle")
    if prm.equations == 3:
        eq_(l2.rev, rc["rev"], "eddy viscosity")
