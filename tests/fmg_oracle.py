"""The oracle on a coarse GROUND level of the full-multigrid start-up (src/solver/solvers.F90:63-117), composed from the
oracle's existing entry points.  The oracle knows two kinds of level: `level` <= 1 runs the fine-grid routines (second
halos, eddy viscosity, directionally scaled radii, cfl, spaceDiscr), `level` > 1 the coarse-level branches of a level
above the ground level.  A block on a ground level g > 1 is the first kind with the reference's choices put into the
parameters and the level flag of each call:

* blocketteRes (the full residual that starts the ground level, solvers.F90:1014-1018): spaceDiscr on every level,
  directional scaling always (blockette.F90:637-653, :1941);
* residual_block (every residual of the smoothers and of multigrid): discr = spaceDiscrCoarse since currentLevel /= 1,
  fine-grid routine since currentLevel == groundLevel (residuals.F90:71-75); currentCfl = cflCoarse (smoothers.F90:138);
* timeStep_block: radiiNeeded = radiiNeededFine = (spaceDiscr == scalar dissipation), an only-radii call returns at once
  otherwise; doScaling = dirScaling, off unless spaceDiscr is scalar dissipation (solverUtils.F90:90-106,
  inputParamRoutines.F90:2824-2833) -- the oracle's level > 1 branch is the unscaled time step.

Pinned bit for bit against the reference's own routines in tests/test_oracle_vs_reference_fmg.py."""
import ctypes as C

import numpy as np

from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
from oracle.pyoracle import Oracle

SCALAR = 1


def _oracle(hb, prm, level):
    o = Oracle(hb, prm)
    o.ob.level = level
    return o


class Ground:
    """the oracle on block `hb` while its level is the ground level (> 1)"""

    def __init__(self, hb, prm):
        self.hb, self.prm = hb, prm
        g = type(prm).from_buffer_copy(prm)
        g.spaceDiscr = prm.spaceDiscrCoarse
        g.cfl = prm.cflCoarse
        self.gprm = g

    def block(self):
        """Oracle for the block path: fine-grid routines of spaceDiscrCoarse with cflCoarse"""
        return _oracle(self.hb, self.gprm, 1)

    def preamble(self):
        """blocketteRes before its core: p, rlv, rev of the owned cells, turbulence and flow BCs, owned-cell rho*E"""
        o = _oracle(self.hb, self.prm, 1)
        o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        d = self.hb.d
        o.L.orc_etot(C.byref(o.ob), C.byref(self.prm), 2, d.il, 2, d.jl, 2, d.kl)

    def blockette_residual(self):
        """the core of blocketteRes in spaceDiscr; it leaves the block's fw alone"""
        fw = self.hb.fw.copy()
        _oracle(self.hb, self.prm, 1).residual_core(RES_FLOW | RES_TURB)
        self.hb.fw[...] = fw

    def time_step(self, only_radii=False):
        scalar = self.prm.spaceDiscr == SCALAR
        if only_radii and not scalar:
            return
        _oracle(self.hb, self.gprm, 1 if scalar else 2).time_step(not only_radii)

    def start(self):
        """solveState on the ground level: the full residual, then timeStep(.false.)"""
        self.blockette_residual()
        self.time_step()


def transfer_to_coarse(prm, ground, coarse):
    """transferToCoarseGrid from the ground level `ground` (a Ground) to the HostBlock `coarse` above it"""
    ground.time_step(only_radii=True)
    of = ground.block()
    of.residual_block(prm.cdisRK[0])
    oc = Oracle(coarse, prm)
    oc.mg_restrict(of)
    oc.apply_flow_bc(False)
    oc.time_step(True)
    oc.mg_store_w1()
    oc.residual_block_coarse(prm.cdisRK[0], init=0)
    oc.mg_forcing()


def mg_cycle(prm, levels, cycling, dadi=False):
    """executeMGCycle (multiGrid.F90:825-955) on the ground level levels[0] (> 1) over `levels`; DADISmoother takes one
    step on every level when the ground level is not 1 (smoothers.F90:400)"""
    g = Ground(levels[0], prm)
    lv = 0
    for n, c in enumerate(cycling):
        if c == -1:
            lv -= 1
            oc = Oracle(levels[lv + 1], prm)
            of = g.block() if lv == 0 else Oracle(levels[lv], prm)
            of.mg_prolong(oc)
            of.apply_flow_bc(lv == 0)
        elif c == 0:
            if lv == 0:
                if n > 0 and cycling[n - 1] != 1:
                    g.time_step()
                    g.block().residual_block(prm.cdisRK[0])
                o = g.block()
            else:
                o = Oracle(levels[lv], prm)
                if n > 0 and cycling[n - 1] != 1:
                    o.time_step(True)
                    o.residual_block(prm.cdisRK[0])
            if dadi:
                o.dadi_step()
            else:
                o.rk_smoother()
        else:
            if lv == 0:
                transfer_to_coarse(prm, g, levels[1])
            else:
                from test_mg_gpu import oracle_transfer_to_coarse
                oracle_transfer_to_coarse(prm, levels[lv], levels[lv + 1])
            lv += 1
    if prm.equations == 3:
        for _ in range(prm.nSubiterTurb):
            g.block().sa_block()
    g.time_step()
    g.block().residual_block(prm.cdisRK[0])


def prolong_solution(prm, fine, coarse):
    """transferToFineGrid(.false.) from the ground level `coarse` to `fine` below it (fine-grid BCs, second halos)"""
    of = _oracle(fine, prm, 1)
    of.mg_prolong_solution(_oracle(coarse, prm, 1))
    of.apply_turb_bc(True)
    of.apply_flow_bc(True); of.apply_flow_bc(True); of.apply_flow_bc(True)


def full_multigrid_start_up(prm, levels, start, n_cycles, cycle, dadi=False):
    """the solver loop `do groundLevel = mgStartlevel, 1, -1` down to ground level 2 on one block per level; returns the
    state (w, p) of every ground level after its cycles"""
    snaps = {}
    for ground, spec in ADFLOW_B200.fmgSchedule(start, cycle):
        g = Ground(levels[ground - 1], prm)
        g.preamble()
        g.start()
        for _ in range(n_cycles):
            mg_cycle(prm, levels[ground - 1:], ADFLOW_B200.cycleStrategy(spec), dadi)
        snaps[ground] = (np.copy(g.hb.w), np.copy(g.hb.p))
        prolong_solution(prm, levels[ground - 2], g.hb)
    return snaps
