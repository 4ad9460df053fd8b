"""The full-multigrid start-up on the device (ADFLOW_B200.fullMultigridStartUp: adfb_set_ground_level, the full residual
and time step that start every ground level, adfb_mg_cycle on the levels at and below it, adfb_mg_prolong_solution) with
a coarse discretisation other than the fine one, against the oracle composition of tests/fmg_oracle.py.  That composition
is pinned bit for bit against the reference's own routines on a coarse ground level in tests/test_oracle_vs_reference_fmg.py.
Tolerances as in test_mg_gpu.py::test_full_multigrid_start_up (1e-9 on states) and
test_multigrid_accelerates_convergence_like_the_oracle (1e-7 on the residual-norm history)."""
import ctypes as C

import numpy as np
import pytest

from adflow_b200 import synthetic as syn
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
from oracle.pyoracle import Oracle

import fmg_oracle as fo
from test_mg_gpu import device, make_levels, oracle_mg_cycle, oracle_transfer_to_coarse
from util import rel_max

pytestmark = pytest.mark.gpu

SC, MA, UP = "central plus scalar dissipation", "central plus matrix dissipation", "upwind"
PAIRS = ([("Euler", f, c) for f in (SC, MA, UP) for c in (SC, MA, UP) if f != c]
         + [(eq, f, SC) for eq in ("laminar NS", "RANS") for f in (MA, UP)])
SHORT = {SC: "scalar", MA: "matrix", UP: "upwind"}
IDS = ["%s-%s-%s" % (eq.split()[0], SHORT[f], SHORT[c]) for eq, f, c in PAIRS]
DADI_SUB = 2   # DADI sub-iterations on ground level 1; a coarse ground level takes one step whatever is asked


def level1_start(prm, hb):
    """solveState on ground level 1: blocketteRes (preamble and core; it leaves the block's fw alone), timeStep(.false.)"""
    o = Oracle(hb, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    fw = hb.fw.copy()
    o.residual_core(RES_FLOW | RES_TURB)
    hb.fw[...] = fw
    o.time_step(True)


def start_levels(options, shape=(16, 12, 8)):
    """three levels with coarse start solutions (restrictions of the fine state) and halos"""
    prm, levels = make_levels(shape, options, 3)
    oracle_transfer_to_coarse(prm, levels[0], levels[1])
    oracle_transfer_to_coarse(prm, levels[1], levels[2])
    for hb in levels:
        hb.fw[...] = 0
    return prm, levels


def run_start_up(options, cycle, smoother, n_after=5):
    prm, levels = start_levels(options)
    dev_levels = [hb.copy() for hb in levels]
    dadi = smoother == "DADI"
    n_cycles = 2
    snaps = fo.full_multigrid_start_up(prm, levels, 3, n_cycles, cycle, dadi)
    fine = levels[0]
    w_start, p_start = fine.w.copy(), fine.p.copy()
    # then cycles on ground level 1, started like solveState
    cyc = ADFLOW_B200.cycleStrategy("3w")
    level1_start(prm, fine)
    ref = [Oracle(fine, prm).norms()[0]]
    for _ in range(n_after):
        oracle_mg_cycle(prm, levels, cyc, dadi_subiter=DADI_SUB if dadi else 0)
        ref.append(Oracle(fine, prm).norms()[0])

    s = device(prm, dev_levels)
    got_snaps = {}
    try:
        prolong = s.mgProlongSolution

        def spy(fine_level=1):   # the ground level fine_level + 1 (block id fine_level) after its cycles
            w, p = s.downloadState(fine_level)[:2]
            got_snaps[fine_level + 1] = (w, p)
            prolong(fine_level)

        s.mgProlongSolution = spy
        s.fullMultigridStartUp(3, n_cycles, cycle, smoother, DADI_SUB)
        assert s.L.adfb_get_ground_level() == 1
        w, p = s.downloadState(0)[:2]
        s.residual(RES_FLOW | RES_TURB)
        s.timeStep(False)
        got = [s.getResNorms()[0]]
        for _ in range(n_after):
            s.mgCycle(cyc, smoother, DADI_SUB)
            got.append(s.getResNorms()[0])
    finally:
        s.close()
    assert sorted(got_snaps) == sorted(snaps) == [2, 3]
    for ground in (3, 2):
        (wd, pd), (wo, po) = got_snaps[ground], snaps[ground]
        assert rel_max(wd, wo) < 1e-9, ("ground level %d state after its cycles" % ground, rel_max(wd, wo))
        assert rel_max(pd, po) < 1e-9, ("ground level %d p" % ground, rel_max(pd, po))
    assert rel_max(w, w_start) < 1e-9, ("fine state after the start-up", rel_max(w, w_start))
    assert rel_max(p, p_start) < 1e-9
    ref, got = np.sqrt(ref), np.sqrt(got)
    assert np.allclose(got, ref, rtol=1e-7, atol=0), ("residual-norm history on level 1", np.abs(got / ref - 1).max())


@pytest.mark.parametrize("smoother", ["RK", "DADI"])
@pytest.mark.parametrize("cycle", ["3w", "3v"])
@pytest.mark.parametrize("eqn,fdisc,cdisc", PAIRS, ids=IDS)
def test_full_multigrid_start_up_with_a_coarse_discretisation(cuda_lib, eqn, fdisc, cdisc, cycle, smoother):
    """fullMultigridStartUp(mgStartlevel = 3, nCyclesCoarse = 2): single-grid cycles on ground level 3, 2-level cycles on
    ground level 2, each ground level started by the full residual in spaceDiscr and timeStep(.false.); then five 3W
    cycles on level 1"""
    run_start_up({"equationType": eqn, "discretization": fdisc, "coarseDiscretization": cdisc}, cycle, smoother)


def test_full_multigrid_start_up_with_equal_discretisations(cuda_lib):
    """the host path of the start-up when both discretisations are the same (RANS, scalar dissipation)"""
    run_start_up(None, "3w", "RK")


def test_two_block_ground_level_with_halo_exchange(cuda_lib):
    """two blocks per level on one device; ground level 2 exchanges second halos after every RK stage and in the
    full residual that starts it"""
    from adflow_b200 import make_params
    from adflow_b200.halo import BlockGrid, build_cartesian_pattern, comm_vars, exchange_numpy, make_grid_blocks

    prm = make_params({"equationType": "laminar NS", "discretization": MA, "nRKStages": 3, "resAveraging": "never"})
    gf = BlockGrid((2, 1, 1), (8, 8, 6), nranks=1)
    fine = make_grid_blocks(gf, 0, prm)
    pf = build_cartesian_pattern(gf, 0)
    vars_ = lambda hb: comm_vars(hb, 1, 5, True, True, True, False)  # noqa: E731
    for hb in fine:
        Oracle(hb, prm).apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)
    coarse = [syn.make_coarse_block(hb, prm) for hb in fine]
    pc = build_cartesian_pattern(BlockGrid((2, 1, 1), (4, 4, 3), nranks=1), 0)
    for f, c in zip(fine, coarse):
        oracle_transfer_to_coarse(prm, f, c)
    exchange_numpy(coarse, pc, vars_)
    for hb in fine + coarse:
        hb.fw[...] = 0
    dev_f, dev_c = [b.copy() for b in fine], [b.copy() for b in coarse]
    n_cycles = 2

    ground = [fo.Ground(c, prm) for c in coarse]
    for g in ground:
        g.preamble()
    exchange_numpy(coarse, pc, vars_)
    for g in ground:
        g.start()
    c0 = [c.w.copy() for c in coarse]
    for _ in range(n_cycles):   # executeMGCycle with the single-grid strategy on ground level 2
        for hb in coarse:
            np.copyto(hb.wn, hb.w[..., :5]); np.copyto(hb.pn, hb.p)
        for st in range(1, prm.nRKStages + 1):
            for g in ground:
                g.block().rk_stage(st)
            exchange_numpy(coarse, pc, vars_)
            if st < prm.nRKStages:
                for g in ground:
                    g.block().residual_block(prm.cdisRK[st])
        for g in ground:
            g.time_step(); g.block().residual_block(prm.cdisRK[0])
    snaps = [(c.w.copy(), c.p.copy()) for c in coarse]
    for f, c in zip(fine, coarse):
        of = Oracle(f, prm)
        of.mg_prolong_solution(Oracle(c, prm))
        of.apply_flow_bc(True); of.apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)
    for f in fine:
        Oracle(f, prm).apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)

    s = ADFLOW_B200(prm)
    got = {}
    try:
        for hb in dev_f:
            s.addBlock(hb)
        for q, hb in enumerate(dev_c):
            s.addCoarseBlock(hb, q)
        s.setCommPattern(pf, level=1)
        s.setCommPattern(pc, level=2, block_offset=2)
        prolong = s.mgProlongSolution

        def spy(fine_level=1):
            got["coarse"] = [s.downloadState(2 + q)[:2] for q in range(2)]
            prolong(fine_level)

        s.mgProlongSolution = spy
        s.fullMultigridStartUp(2, n_cycles, "2v")
        got["fine"] = [s.downloadState(q)[:2] for q in range(2)]
    finally:
        s.close()
    for q in range(2):
        wd, pd = got["coarse"][q]
        assert np.abs(snaps[q][0][coarse[q].d.owned()] - c0[q][coarse[q].d.owned()]).max() > 0
        assert rel_max(wd[..., :5], snaps[q][0][..., :5]) < 1e-9, ("ground level 2, block", q, rel_max(wd[..., :5], snaps[q][0][..., :5]))
        assert rel_max(pd, snaps[q][1]) < 1e-9
        wf, pf_ = got["fine"][q]
        assert rel_max(wf[..., :5], fine[q].w[..., :5]) < 1e-9, ("fine block after the start-up", q, rel_max(wf[..., :5], fine[q].w[..., :5]))
        assert rel_max(pf_, fine[q].p) < 1e-9
