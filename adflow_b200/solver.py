"""Host-side mirror of the pyADflow calls that sit on the hot path.

``ADFLOW_B200`` keeps the names, argument meaning and ordering conventions of
``adflow/pyADflow.py`` for the calls that reach the per-block numerics
(``getResidual`` :5359, ``getStates`` :5174, ``setStates`` :5181,
``getFreeStreamResidual`` :5422, ``getResNorms`` :3399) and routes them through
the C ABI (``include/adflow_b200.h``) to the CUDA kernels -- the same calls the
Fortran drivers would make through ISO_C_BINDING (INTEGRATION.md).  It is a thin
layer: all arithmetic happens on the device; there is no CPU path.

State/residual vectors use the reference ordering (``NKSolvers.F90:1240-1255``):
for each block, k, j, i, then the nw variables of the cell (AoS per cell).
"""
import ctypes as C
import math
import time

import numpy as np

from . import _lib
from ._lib import AdfbSubface, check, ptr

RES_DISS_APPROX, RES_VISC_APPROX, RES_UPDATE_INTERMED = 1, 2, 4
RES_FLOW, RES_TURB, RES_STORE_WALL, RES_SKIP_PREAMBLE = 8, 16, 32, 64

# adfb_monitor: `what` bits and the entries of its out[10]
MON_SUMS, MON_MAXIMA = 1, 2
# the monitored quantities of convergenceInfo by their CGNS names (cgnsNames.f90), in the order checkMonitor sorts them
# (inputParamRoutines.F90:120-330), with their entry of adfb_monitor's out[]
MONITOR_SLOTS = {"RSDMassRMS": 0, "RSDMomentumXRMS": 1, "RSDMomentumYRMS": 2, "RSDMomentumZRMS": 3,
                 "RSDEnergyStagnationDensityRMS": 4, "RSDTurbulentSANuTildeRMS": 5, "totalR": 6, "MaxDiffHAndHinf": 7,
                 "MaxMach": 8, "MaxRatioEddyAndLaminarViscosity": 9}
# the keywords of the pyADflow option monitorVariables (monitorVariables, inputParamRoutines.F90:1480-1660)
_MONITOR_KEYWORDS = {"resrho": ["RSDMassRMS"], "resmom": ["RSDMomentumXRMS", "RSDMomentumYRMS", "RSDMomentumZRMS"],
                     "resrhoe": ["RSDEnergyStagnationDensityRMS"], "resturb": ["RSDTurbulentSANuTildeRMS"],
                     "totalr": ["totalR"], "hdiff": ["MaxDiffHAndHinf"], "mach": ["MaxMach"],
                     "eddyv": ["MaxRatioEddyAndLaminarViscosity"]}
_FORCE_MONITORS = ("cl", "clp", "clv", "cd", "cdp", "cdv", "cfx", "cfy", "cfz", "cmx", "cmy", "cmz")
_SOLUTION_MONITORS = ("yplus", "sepsensor", "sepsensorksarea", "cavitation", "axismoment")
# pyADflow's default monitorVariables without the force monitors cl and cd, which the device does not monitor
DEFAULT_MONITOR_VARIABLES = ("cpu", "resrho", "resturb")


def monitor_names(variables, rans):
    """The CGNS names convergenceInfo monitors for the monitorVariables keywords `variables`, in its order, and whether
    "cpu" (the host wall time) was asked for.  resrho and totalR are always monitored; resturb and eddyv only with RANS
    (checkMonitor drops them otherwise).  The force and getSolution monitors are refused with a ValueError."""
    names, cpu = {"RSDMassRMS", "totalR"}, False
    for v in variables:
        key = v.lower()
        if key == "cpu":
            cpu = True
        elif key in _FORCE_MONITORS:
            raise ValueError("monitor variable %r is a force or moment coefficient, which the device does not monitor: "
                             "evaluate it with evalFunctions after residual(... | RES_STORE_WALL)" % v)
        elif key in _SOLUTION_MONITORS:
            raise ValueError("monitor variable %r is a getSolution quantity, which the device does not evaluate" % v)
        elif key not in _MONITOR_KEYWORDS:
            raise ValueError("unknown monitor variable %r; known: cpu, %s" % (v, ", ".join(sorted(_MONITOR_KEYWORDS))))
        elif rans or key not in ("resturb", "eddyv"):
            names.update(_MONITOR_KEYWORDS[key])
    return [n for n in MONITOR_SLOTS if n in names], cpu


def convergence_status(ground_level, approx_total_its, n_cycles, values, rho_res, rho_res_start, total_r, total_r0,
                       total_r_start, L2Convergence=1e-8, L2ConvergenceCoarse=1e-2, L2ConvergenceRel=1e-16,
                       maxL2DeviationFactor=1.0):
    """(converged, failed) after one convergenceInfo of the steady solveState (solvers.F90:1726-1763, 1873-1920): above
    ground level 1 rhoRes < L2ConvergenceCoarse rhoResStart; on level 1 totalR < L2Convergence totalR0 or
    totalR < L2ConvergenceRel totalRStart.  Failed: a NaN among the monitored `values`, or on ground level 1 with the
    nCycles cycles spent, totalR > maxL2DeviationFactor totalR0 L2Convergence."""
    if ground_level != 1:
        converged = rho_res < L2ConvergenceCoarse * rho_res_start
    else:
        converged = total_r < L2Convergence * total_r0 or total_r < L2ConvergenceRel * total_r_start
    failed = any(math.isnan(v) for v in values)
    if not failed and ground_level == 1 and approx_total_its >= n_cycles:
        failed = total_r > maxL2DeviationFactor * total_r0 * L2Convergence
    return bool(converged), bool(failed)


class ADFLOW_B200:
    def __init__(self, prm, device=0, rank=0, nranks=1, unique_id=None):
        self.L = _lib.load()
        check(self.L.adfb_init(device, unique_id, rank, nranks), "adfb_init")
        self.prm = prm
        self.nranks = nranks
        check(self.L.adfb_set_params(C.byref(prm)), "adfb_set_params")
        self.blocks = []  # HostBlock descriptors (extents only are needed after upload)
        self.blockLevels = []
        self._keep = []
        # nCellGlobal(level): the owned cells of a level over all ranks.  Formed from this rank's blocks on one rank; a
        # multi-rank host sets it for each level it monitors.
        self.nCellGlobal = {}
        self.totalR0 = None   # getFreeStreamResidual's value, once per flow (freeStreamResSet)
        self._totalR = 0.0    # the totalR last passed to setTotalResiduals

    # -- data model ---------------------------------------------------------
    def addBlock(self, hb, level=1, upload_metrics=True):
        """Create the device mirror of one block and upload geometry + BC data + state."""
        blk = len(self.blocks)
        d = hb.d
        check(self.L.adfb_block_create(blk, level, d.nx, d.ny, d.nz, hb.nw, int(hb.right_handed)), "adfb_block_create")
        self.setGeometry(blk, hb, upload_metrics)
        if hb.subfaces:
            self.setBCData(blk, hb.subfaces)
        self.blocks.append(hb)
        self.blockLevels.append(level)
        self.uploadState(blk, hb)
        return blk

    def setGeometry(self, blk, hb, upload_metrics=True):
        """Upload the geometry of hb to block blk (a mesh warp on a live block); upload_metrics=False: the face
        metrics are formed from the coordinates on the device."""
        r = hb.ref
        si = r("si") if upload_metrics else None
        sj = r("sj") if upload_metrics else None
        sk = r("sk") if upload_metrics else None
        arrs = [r("x"), si, sj, sk, r("vol"), r("volRef"), r("d2Wall"), r("porI"), r("porJ"), r("porK"), r("iblank")]
        check(self.L.adfb_block_set_geometry(blk, *[ptr(a) for a in arrs]), "adfb_block_set_geometry")

    def setBCData(self, blk, subfaces):
        """Replace the subfaces of block blk (layout and prescribed BC data)."""
        n = len(subfaces)
        sf = (AdfbSubface * max(n, 1))()
        keep = []
        for q, s in enumerate(subfaces):
            sf[q].bcType, sf[q].faceId = s["bcType"], s["faceId"]
            sf[q].icBeg, sf[q].icEnd, sf[q].jcBeg, sf[q].jcEnd = s["icBeg"], s["icEnd"], s["jcBeg"], s["jcEnd"]
            sf[q].subsonicInletTreatment = int(s.get("subsonicInletTreatment", 0))
            for name in ("norm", "rface", "uSlip", "TNSWall", "ps", "rho", "velx", "vely", "velz", "ptInlet", "ttInlet", "htInlet",
                         "flowXdirInlet", "flowYdirInlet", "flowZdirInlet", "turbInlet"):
                a = s.get(name)
                if a is not None:
                    a = np.asfortranarray(a, dtype=np.float64)
                    keep.append(a)
                    setattr(sf[q], name, a.ctypes.data)
            if s.get("iblank") is not None:   # BCData%iblank, int32 (icBeg:icEnd, jcBeg:jcEnd)
                a = np.asfortranarray(s["iblank"], dtype=np.int32)
                if a.shape != (s["icEnd"] - s["icBeg"] + 1, s["jcEnd"] - s["jcBeg"] + 1):
                    raise ValueError("subface %d: iblank has shape %s, not the subface's cell range" % (q, a.shape))
                keep.append(a)
                sf[q].iblank = a.ctypes.data
        check(self.L.adfb_block_set_bc(blk, n, sf), "adfb_block_set_bc")

    def uploadState(self, blk, hb, with_visc=True):
        check(self.L.adfb_upload_state(blk, ptr(hb.w), ptr(hb.p)), "adfb_upload_state")
        if with_visc:
            check(self.L.adfb_upload_visc(blk, ptr(hb.rlv), ptr(hb.rev)), "adfb_upload_visc")

    def setParams(self, prm):
        self.prm = prm
        check(self.L.adfb_set_params(C.byref(prm)), "adfb_set_params")

    # -- hot path -----------------------------------------------------------
    def residual(self, flags=RES_FLOW | RES_TURB, level=1):
        """blocketteRes (src/NKSolver/blockette.F90:70-297) on all local blocks."""
        check(self.L.adfb_residual(level, flags), "adfb_residual")

    def setCommPattern(self, pat, level=1, block_offset=0):
        """Upload the 1-to-1 communication pattern of one grid level (adflow_b200.halo.build_cartesian_pattern).
        block_offset: added to the pattern's local block indices (device ids of a coarse level's blocks follow the
        finer levels')."""
        a = {k: np.ascontiguousarray(v, dtype=np.int32).copy() for k, v in pat.items()}
        if block_offset:
            for k in ("sendList", "recvList", "donorList", "haloList"):
                if a[k].size:
                    a[k][:, 0] += block_offset
        self._keep.append(a)
        p = lambda x: x.ctypes.data if x.size else None  # noqa: E731
        check(self.L.adfb_comm_set_pattern(level, len(a["nbrRank"]), p(a["nbrRank"]), p(a["sendCount"]), p(a["recvCount"]),
                                           p(a["sendList"]), p(a["recvList"]), len(a["donorList"]), p(a["donorList"]),
                                           p(a["haloList"])), "adfb_comm_set_pattern")

    def setOversetPattern(self, pat, level=1):
        """Upload an overset (interpolating) communication pattern: the keys of setCommPattern plus the
        8 weights per donor entry in "sendInterp" / "donorInterp" (adflow_b200.halo.build_overset_pattern)."""
        a = {k: np.ascontiguousarray(v, dtype=(np.float64 if k.endswith("Interp") else np.int32)) for k, v in pat.items()}
        self._keep.append(a)
        p = lambda x: x.ctypes.data if x.size else None  # noqa: E731
        check(self.L.adfb_comm_set_overset(level, len(a["nbrRank"]), p(a["nbrRank"]), p(a["sendCount"]), p(a["recvCount"]),
                                           p(a["sendList"]), p(a["sendInterp"]), p(a["recvList"]), len(a["donorList"]),
                                           p(a["donorList"]), p(a["donorInterp"]), p(a["haloList"])), "adfb_comm_set_overset")

    def setOrphans(self, blk, orphans, mu_inf, eddy_vis_inf_ratio):
        """orphans(3, nOrphans) of one block (cell indices with the reference's bounds) and the free-stream viscosities
        orphanAverage falls back to; every exchange then ends with orphanAverage on that block."""
        a = np.ascontiguousarray(np.asarray(orphans, dtype=np.int32).reshape(-1, 3))
        check(self.L.adfb_block_set_orphans(blk, len(a), a.ctypes.data_as(C.c_void_p) if len(a) else None, C.c_double(mu_inf),
                                            C.c_double(eddy_vis_inf_ratio)), "adfb_block_set_orphans")

    def haloExchange(self, start=1, end=None, comm_pressure=True, comm_gamma=True, comm_viscous=True, level=1):
        """whalo2(level, start, end, commPressure, commGamma, commViscous)."""
        if end is None:
            end = self.blocks[0].nw
        check(self.L.adfb_halo_exchange(level, start, end, int(comm_pressure), int(comm_gamma), int(comm_viscous)),
              "adfb_halo_exchange")

    def applyBCs(self, second_halo=True, with_turb=True, level=1):
        """applyAllBC (+ turbulence halo treatment) on all local blocks."""
        check(self.L.adfb_apply_bcs(level, int(second_halo), int(with_turb)), "adfb_apply_bcs")

    def timeStep(self, only_radii=False, level=1):
        check(self.L.adfb_timestep(level, int(only_radii)), "adfb_timestep")

    def smootherResidual(self, rk_stage=0, level=1):
        """initres + residual of the smoother loops; rFil = cdisRK(rk_stage+1)."""
        check(self.L.adfb_smoother_residual(level, rk_stage), "adfb_smoother_residual")

    def rkStage(self, stage, level=1):
        check(self.L.adfb_rk_stage(level, stage), "adfb_rk_stage")

    def rkCycle(self, level=1):
        """RungeKuttaSmoother (src/solver/smoothers.F90:4)."""
        check(self.L.adfb_rk_cycle(level), "adfb_rk_cycle")

    def dadiStep(self, level=1):
        """executeDADIStep (src/solver/smoothers.F90:425)."""
        check(self.L.adfb_dadi_step(level), "adfb_dadi_step")

    def dadiCycle(self, n_subiterations=1, level=1):
        """DADISmoother (src/solver/smoothers.F90:383)."""
        check(self.L.adfb_dadi_cycle(level, n_subiterations), "adfb_dadi_cycle")

    # -- ANK pieces (module ANKSolver, src/NKSolver/NKSolvers.F90) ----------------------------------------------
    def ankSetParams(self, ank):
        self._ank = ank
        check(self.L.adfb_ank_set_params(C.byref(ank)), "adfb_ank_set_params")

    def ankTimeStepMat(self):
        """computeTimeStepMat: blocks from the current state and dtl (call timeStep / a residual with
        RES_UPDATE_INTERMED first)"""
        check(self.L.adfb_ank_time_step_mat(), "adfb_ank_time_step_mat")

    def ankVecSize(self):
        ns = lambda hb: hb.nw if self._ank.coupled else 5  # noqa: E731
        return sum(hb.d.ncells * ns(hb) for hb in self.blocks if getattr(hb, "level", 1) == 1)

    def ankFormFunction(self, in_vec):
        v = np.ascontiguousarray(in_vec, dtype=np.float64)
        r = np.empty_like(v)
        check(self.L.adfb_ank_form_function(v.ctypes.data, r.ctypes.data, v.size), "adfb_ank_form_function")
        return r

    def ankMffdSetBase(self, U):
        U = np.ascontiguousarray(U, dtype=np.float64)
        check(self.L.adfb_ank_mffd_set_base(U.ctypes.data, U.size), "adfb_ank_mffd_set_base")

    def ankMffdApply(self, a, h=-1.0):
        a = np.ascontiguousarray(a, dtype=np.float64)
        y = np.empty_like(a)
        check(self.L.adfb_ank_mffd_apply(a.ctypes.data, y.ctypes.data, a.size, h), "adfb_ank_mffd_apply")
        return y

    def ankMffdApplyDevice(self, a_ptr, y_ptr, n, h=-1.0):
        check(self.L.adfb_ank_mffd_apply_device(a_ptr, y_ptr, n, h), "adfb_ank_mffd_apply_device")

    def gmresSolve(self, rhs, op="ANK", restart=30, max_its=60, rtol=1e-6, atol=1e-50):
        """right-preconditioned restarted GMRES on the device (identity preconditioner) for the NK or ANK product;
        returns (x, iterations, residual norm estimate)"""
        b = np.ascontiguousarray(rhs, dtype=np.float64)
        x = np.zeros_like(b)
        its, rn = C.c_int(0), C.c_double(0.0)
        check(self.L.adfb_gmres_solve({"NK": 0, "ANK": 1, "TSMAT": 2}[op], b.ctypes.data, x.ctypes.data, b.size, restart, max_its, rtol, atol,
                                      None, None, C.byref(its), C.byref(rn)), "adfb_gmres_solve")
        return x, its.value, rn.value

    def ankPhysicalityCheck(self, w_vec, delta_w, lambda_p=1.0):
        """returns (lambdaP, deltaW) -- deltaW with the clipped turbulence updates (coupled ANK)"""
        w = np.ascontiguousarray(w_vec, dtype=np.float64)
        dv = np.array(delta_w, dtype=np.float64, order="C", copy=True)
        lam = C.c_double(lambda_p)
        check(self.L.adfb_ank_physicality_check(w.ctypes.data, dv.ctypes.data, w.size, C.byref(lam)), "adfb_ank_physicality_check")
        return lam.value, dv

    # turbulence KSP of the decoupled ANK: one turbulence variable per owned cell
    def ankFormFunctionTurb(self, in_vec):
        """FormFunction_mf_turb (NKSolvers.F90:2540-2612)"""
        v = np.ascontiguousarray(in_vec, dtype=np.float64)
        r = np.empty_like(v)
        check(self.L.adfb_ank_form_function_turb(v.ctypes.data, r.ctypes.data, v.size), "adfb_ank_form_function_turb")
        return r

    def ankMffdTurbSetBase(self, U):
        U = np.ascontiguousarray(U, dtype=np.float64)
        check(self.L.adfb_ank_mffd_turb_set_base(U.ctypes.data, U.size), "adfb_ank_mffd_turb_set_base")

    def ankMffdTurbApply(self, a, h):
        a = np.ascontiguousarray(a, dtype=np.float64)
        y = np.empty_like(a)
        check(self.L.adfb_ank_mffd_turb_apply(a.ctypes.data, y.ctypes.data, a.size, C.c_double(h)), "adfb_ank_mffd_turb_apply")
        return y

    def ankPhysicalityCheckTurb(self, w_vec, delta_w, lambda_p=1.0):
        """physicalityCheckANKTurb (NKSolvers.F90:3212-3335): returns (lambdaP, deltaW with the clipped updates)"""
        w = np.ascontiguousarray(w_vec, dtype=np.float64)
        dv = np.array(delta_w, dtype=np.float64, order="C", copy=True)
        lam = C.c_double(lambda_p)
        check(self.L.adfb_ank_physicality_check_turb(w.ctypes.data, dv.ctypes.data, w.size, C.byref(lam)), "adfb_ank_physicality_check_turb")
        return lam.value, dv

    # -- multigrid (src/solver/multiGrid.F90) ----------------------------------------------------------------
    def addCoarseBlock(self, coarse_hb, fine_blk):
        """Device mirror of the next coarser level of block `fine_blk` + the transfer tables (createCoarseBlocks,
        src/preprocessing/coarseUtils.F90): coarse_hb.mg holds mg?Fine / mg?Weight, the fine HostBlock's mg holds
        mg?Coarse (see synthetic.make_coarse_block).  Returns the coarse block id."""
        fine_hb = self.blocks[fine_blk]
        blk = self.addBlock(coarse_hb, level=coarse_hb.level)
        dc, df = coarse_hb.d, fine_hb.d
        f = np.asfortranarray
        tabs = []
        for nm, e in zip("IJK", (dc.ie, dc.je, dc.ke)):
            tabs.append(f(coarse_hb.mg["mg%sFine" % nm][1:e + 1, :].astype(np.int32)))
        for nm, l in zip("IJK", (dc.il, dc.jl, dc.kl)):
            tabs.append(np.ascontiguousarray(coarse_hb.mg["mg%sWeight" % nm][2:l + 1], dtype=np.float64))
        for nm, l in zip("IJK", (df.il, df.jl, df.kl)):
            tabs.append(f(fine_hb.mg["mg%sCoarse" % nm][2:l + 1, :].astype(np.int32)))
        check(self.L.adfb_block_set_mg(blk, fine_blk, *[t.ctypes.data for t in tabs]), "adfb_block_set_mg")
        return blk

    def mgRestrict(self, fine_level=1):
        """transferToCoarseGrid from fine_level to fine_level + 1"""
        check(self.L.adfb_mg_restrict(fine_level), "adfb_mg_restrict")

    def mgProlong(self, fine_level=1):
        """transferToFineGrid(corrections=.true.) from fine_level + 1 to fine_level"""
        check(self.L.adfb_mg_prolong(fine_level), "adfb_mg_prolong")

    def setGroundLevel(self, level):
        """iteration%groundLevel (solvers.F90:63): the finest level of the multigrid cycles that follow"""
        check(self.L.adfb_set_ground_level(level), "adfb_set_ground_level")

    def mgProlongSolution(self, fine_level=1):
        """transferToFineGrid(corrections=.false.): the solution of ground level fine_level + 1 -> fine_level"""
        check(self.L.adfb_mg_prolong_solution(fine_level), "adfb_mg_prolong_solution")

    @staticmethod
    def fmgSchedule(mg_start_level, cycle="sg"):
        """Ground levels of the full-multigrid start-up with the cycle each of them runs: the strategy of `cycle` ('sg', '<n>v',
        '<n>w') shortened to the levels at and below the ground level (setCycleStrategy works on nMGLevels - groundLevel + 1
        levels, src/solver/multiGrid.F90:957-1030).  Returns [(groundLevel, spec), ...] for groundLevel = mgStartlevel .. 2."""
        n_lev = 1 if cycle.lower() == "sg" else int(cycle[:-1])
        if mg_start_level < 1 or mg_start_level > max(n_lev, 1):
            raise ValueError("mgStartlevel %d outside 1..%d" % (mg_start_level, max(n_lev, 1)))
        out = []
        for ground in range(mg_start_level, 1, -1):
            left = n_lev - ground + 1          # levels ground .. n_lev take part
            out.append((ground, "sg" if left < 2 else "%d%s" % (left, cycle[-1].lower())))
        return out

    def fullMultigridStartUp(self, mg_start_level, n_cycles_coarse, cycle="sg", smoother="RK", n_subiterations=1):
        """The full-multigrid start-up of `solver` (src/solver/solvers.F90:63-117): nCyclesCoarse cycles of executeMGCycle on
        every ground level mgStartlevel, ..., 2 (fmgSchedule), each followed by transferToFineGrid(.false.); leaves the ground
        level at 1.  Each ground level starts like solveState (solvers.F90:1014-1018): the full residual (blocketteRes, in
        spaceDiscr), then timeStep(.false.); the first smoothing step of the first cycle consumes that residual."""
        for ground, spec in self.fmgSchedule(mg_start_level, cycle):
            self.setGroundLevel(ground)
            self.residual(RES_FLOW | RES_TURB, level=ground)
            self.timeStep(False, level=ground)
            cyc = self.cycleStrategy(spec)
            for _ in range(n_cycles_coarse):
                self.mgCycle(cyc, smoother, n_subiterations)
            self.mgProlongSolution(ground - 1)
        self.setGroundLevel(1)

    @staticmethod
    def cycleStrategy(spec):
        """inputIteration%cycleStrategy of the pyADflow option MGCycle ('sg', '2v', '3w', ...), extractMgInfo /
        setEntriesWcycle, src/inputParam/inputParamRoutines.F90:880-945,1127-1180: an n-level V cycle is
        (0 1)^(n-1) (0 -1)^(n-1); a W cycle is 0 1 W(n-1) W(n-1) 0 -1 with W(2) = 0 1 0 -1."""
        spec = spec.lower()
        if spec == "sg":
            return [0]
        n, kind = int(spec[:-1]), spec[-1]
        if n < 2 or kind not in "vw":
            raise ValueError("MGCycle must be sg, <n>v or <n>w with n >= 2")
        if kind == "v":
            return [0, 1] * (n - 1) + [0, -1] * (n - 1)

        def wcyc(levels):
            if levels == 2:
                return [0, 1, 0, -1]
            inner = wcyc(levels - 1)
            return [0, 1] + inner + inner + [0, -1]

        return wcyc(n)

    def mgCycle(self, cycling, smoother="RK", n_subiterations=1):
        """executeMGCycle on ground level 1 with cycling in {-1, 0, +1} (iteration%cycling); smoother "RK" or "DADI" """
        cyc = np.ascontiguousarray(cycling, dtype=np.int32)
        sm = 0 if smoother == "RK" else int(n_subiterations)
        check(self.L.adfb_mg_cycle(len(cyc), cyc.ctypes.data, sm), "adfb_mg_cycle")

    def turbSolveDDADI(self, n_sub_iter_turb=None, level=1):
        """turbSolveDDADI (src/turbulence/turbAPI.F90:4)."""
        n = self.prm.nSubiterTurb if n_sub_iter_turb is None else n_sub_iter_turb
        check(self.L.adfb_sa_ddadi(level, n), "adfb_sa_ddadi")

    def referenceShockSensor(self, level=1):
        """referenceShockSensor (src/adjoint/adjointUtils.F90:1900): freeze the sensor field."""
        check(self.L.adfb_reference_shock_sensor(level), "adfb_reference_shock_sensor")

    def downloadResidual(self, blk):
        hb = self.blocks[blk]
        out = np.zeros(hb.d.box + (hb.nw,), order="F")
        check(self.L.adfb_download_residual(blk, ptr(out)), "adfb_download_residual")
        return out

    def downloadState(self, blk):
        hb = self.blocks[blk]
        w = np.zeros(hb.d.box + (hb.nw,), order="F")
        p, rlv, rev = (np.zeros(hb.d.box, order="F") for _ in range(3))
        check(self.L.adfb_download_state(blk, ptr(w), ptr(p), ptr(rlv), ptr(rev)), "adfb_download_state")
        return w, p, rlv, rev

    def downloadIntermed(self, blk):
        d = self.blocks[blk].d
        shp = (d.ie, d.je, d.ke)
        a = [np.zeros(shp, order="F") for _ in range(4)]
        check(self.L.adfb_download_intermed(blk, *[ptr(x) for x in a]), "adfb_download_intermed")
        return dict(zip(("dtl", "radI", "radJ", "radK"), a))

    def downloadArray(self, blk, name, ncomp=1):
        hb = self.blocks[blk]
        shp = hb.d.box + ((ncomp,) if ncomp > 1 else ())
        out = np.zeros(shp, order="F")
        check(self.L.adfb_download_array(blk, name.encode(), ptr(out)), "adfb_download_array")
        return out

    def getResNorms(self):
        """(sum (dw_rho/vol)^2, sum all (dw/vol)^2) -- getCurrentResidual, NKSolvers.F90:335-370."""
        out = (C.c_double * 2)()
        check(self.L.adfb_norms(out), "adfb_norms")
        return np.array([out[0], out[1]])

    def getFreeStreamResidual(self):
        """totalR0: the L2 norm of the residual of the uniform free stream on the fine grid (pyADflow.py:5422-5425,
        getFreeStreamResidual NKSolvers.F90:280-333); the state on the device is left as it was."""
        out = (C.c_double * 2)()
        check(self.L.adfb_free_stream_residual(out), "adfb_free_stream_residual")
        return float(np.sqrt(out[1]))

    INF_CHANGE_TYPES = {"offset": 0, "rotate": 1}

    def infChangeCorrection(self, old_winf, tol=1e-12, kind="offset"):
        """infChangeCorrection (initializeFlow.F90:191-316, pyADflow.py:3416-3421): correct the state of the level-1 blocks
        from the free stream old_winf (its first five entries) to the wInf of the current parameters (setParams first).
        kind is pyADflow's infChangeCorrectionType, "offset" or "rotate".  Returns whether the state was changed: a change
        whose rho, u, v part is below tol is skipped, as in the reference."""
        if kind not in self.INF_CHANGE_TYPES:
            raise ValueError("infChangeCorrection: kind must be 'offset' or 'rotate', got %r" % (kind,))
        old = (C.c_double * 5)(*[float(v) for v in list(old_winf)[:5]])
        applied = C.c_int(0)
        check(self.L.adfb_inf_change_correction(old, float(tol), self.INF_CHANGE_TYPES[kind], C.byref(applied)),
              "adfb_inf_change_correction")
        return bool(applied.value)

    def setUniformFlow(self, level, mu_inf, eddy_vis_inf_ratio):
        """setUniformFlow (initializeFlow.F90:2143-2212) on the blocks of `level`: w = wInf, dw = fw = 0, p = pInfCorr,
        rlv = mu_inf (viscous), rev = eddy_vis_inf_ratio * mu_inf (RANS), halos included."""
        check(self.L.adfb_set_uniform_flow(level, float(mu_inf), float(eddy_vis_inf_ratio)), "adfb_set_uniform_flow")

    def resetFlow(self, mg_start_level, mu_inf, eddy_vis_inf_ratio):
        """_resetFlow (pyADflow.py:3097-3111): the ground level becomes mgStartLevel and its blocks get the uniform flow;
        fullMultigridStartUp(mg_start_level, ...) or solve(mg_start_level, ...) then starts from there.  The cached
        free-stream residual totalR0 is forgotten (freeStreamResSet = .false.)."""
        self.setGroundLevel(mg_start_level)
        self.setUniformFlow(mg_start_level, mu_inf, eddy_vis_inf_ratio)
        self.totalR0 = None

    def setTotalResiduals(self, totalR, totalR0):
        """iteration%totalR and totalR0, read by the dissipation-based continuation (useDissContinuation)."""
        check(self.L.adfb_set_total_residuals(float(totalR), float(totalR0)), "adfb_set_total_residuals")

    # -- convergence monitor and the steady solver loop (src/solver/solvers.F90) -----------------------------------
    def monitorSums(self, level=1, what=MON_SUMS | MON_MAXIMA):
        """adfb_monitor: the ten all-reduced sums and maxima of the blocks of `level` (include/adflow_b200.h)"""
        out = (C.c_double * 10)()
        check(self.L.adfb_monitor(level, what, out), "adfb_monitor")
        return np.array(list(out))

    def _n_cell_global(self, level):
        if level not in self.nCellGlobal:
            if self.nranks > 1:
                raise ValueError("nCellGlobal[%d] must be set on a multi-rank context" % level)
            self.nCellGlobal[level] = sum(hb.d.nx * hb.d.ny * hb.d.nz for hb, lv in zip(self.blocks, self.blockLevels) if lv == level)
        return self.nCellGlobal[level]

    def _monitor(self, level, names):
        what = MON_SUMS | (MON_MAXIMA if any(MONITOR_SLOTS[n] > 6 for n in names) else 0)
        raw = self.monitorSums(level, what)
        n = float(self._n_cell_global(level))
        out = {}
        for name in names:
            q = MONITOR_SLOTS[name]
            out[name] = math.sqrt(raw[q] / n) if q < 6 else math.sqrt(raw[q]) if q == 6 else float(raw[q])
        return out

    def monitor(self, level=1, names=DEFAULT_MONITOR_VARIABLES):
        """The values convergenceInfo monitors on ground level `level` for the monitorVariables keywords `names`, as it
        finishes them (solvers.F90:1642-1706), by CGNS name: a residual norm is sqrt(sum / nCellGlobal(level)), totalR is
        sqrt(sum), the maxima as they are.  resrho and totalR are always there; "cpu" adds nothing here (solveState
        records the host wall time)."""
        return self._monitor(level, monitor_names(names, self.prm.equations == 3)[0])

    def solveState(self, nCycles=2000, nCyclesCoarse=500, L2Convergence=1e-8, L2ConvergenceCoarse=1e-2, L2ConvergenceRel=1e-16,
                   maxL2DeviationFactor=1.0, MGCycle="sg", smoother="DADI", nSubiter=1, monitorVariables=DEFAULT_MONITOR_VARIABLES):
        """The steady solveState with the smoother on every iteration (solvers.F90:892-1236, neither ANK nor NK) on the
        current ground level; the keyword arguments are the pyADflow options of the same names, with their defaults
        (monitorVariables without cl and cd).  Returns {"converged", "failed", "history"}, the history as
        getConvergenceHistory gives it (pyADflow.py:1404): "total minor iters", "iter type", "CFL", "step",
        "linear res", "wall time" with "cpu", and one list per monitored CGNS name, iteration 0 first."""
        if smoother not in ("DADI", "Runge-Kutta", "RK"):
            raise ValueError("smoother must be 'DADI' or 'Runge-Kutta', got %r" % (smoother,))
        sm = "DADI" if smoother == "DADI" else "RK"
        names, cpu = monitor_names(monitorVariables, self.prm.equations == 3)
        t0 = time.perf_counter()
        ground = int(self.L.adfb_get_ground_level())
        n_mg = nCycles if ground == 1 else nCyclesCoarse
        cyc = self.cycleStrategy(MGCycle if ground == 1 else dict(self.fmgSchedule(ground, MGCycle))[ground])
        if ground == 1 and self.totalR0 is None:
            self.totalR0 = self.getFreeStreamResidual()
        total_r0 = self.totalR0 if self.totalR0 is not None else 0.0
        diss = bool(self.prm.useDissContinuation)
        hist = {"total minor iters": [], "iter type": [], "CFL": [], "step": [], "linear res": []}
        if cpu:
            hist["wall time"] = []
        for name in names:
            hist[name] = []

        def record(its, kind, cfl, step, vals):
            # convergenceInfo stores the CFL and the step only when they are not negative (solvers.F90:1588-1620)
            hist["total minor iters"].append(its)
            hist["iter type"].append(kind)
            hist["CFL"].append(max(cfl, 0.0))
            hist["step"].append(max(step, 0.0))
            hist["linear res"].append(0.0)
            if cpu:
                hist["wall time"].append(time.perf_counter() - t0)
            for name in names:
                hist[name].append(vals[name])
            if diss:
                self._totalR = vals["totalR"]
                self.setTotalResiduals(self._totalR, total_r0)

        def status(its, vals):
            return convergence_status(ground, its, nCycles, [vals[n] for n in names], vals["RSDMassRMS"], rho_start, vals["totalR"],
                                      total_r0, total_r_start, L2Convergence, L2ConvergenceCoarse, L2ConvergenceRel,
                                      maxL2DeviationFactor)

        if diss:   # the first residual reads the new totalR0 and the totalR of the last monitor
            self.setTotalResiduals(self._totalR, total_r0)
        # the first residual (blocketteRes with the store-wall flag, blockette.F90:135), then timeStep(.false.)
        self.residual(RES_FLOW | RES_TURB | RES_STORE_WALL, level=ground)
        self.timeStep(False, level=ground)
        vals = self._monitor(ground, names)
        rho_start, total_r_start = vals["RSDMassRMS"], vals["totalR"]
        record(0, "None", -1.0, -1.0, vals)
        converged, failed = False, any(math.isnan(vals[n]) for n in names)
        its = 0
        cfl = self.prm.cfl if ground == 1 else self.prm.cflCoarse
        while its < n_mg and not failed:
            self.mgCycle(cyc, sm, nSubiter)
            its += 1
            vals = self._monitor(ground, names)
            record(its, sm, cfl, 1.0, vals)
            converged, failed = status(its, vals)
            if converged:
                break
        return {"converged": converged, "failed": failed, "history": hist}

    def solve(self, mg_start_level, **options):
        """The steady `solver` loop (solvers.F90:63-117): solveState(**options) on every ground level mgStartLevel .. 1,
        transferToFineGrid(.false.) between them.  Returns [(groundLevel, result of solveState), ...]."""
        out = []
        for ground in range(mg_start_level, 0, -1):
            self.setGroundLevel(ground)
            out.append((ground, self.solveState(**options)))
            if ground > 1:
                self.mgProlongSolution(ground - 1)
        self.setGroundLevel(1)
        return out

    def getForces(self, ref_point=(0.0, 0.0, 0.0), p_ref=1.0, level=1):
        """Fp, Fv, Mp, Mv (rows) summed over the wall subfaces of all ranks -- wallIntegrationFace,
        src/solver/surfaceIntegrations.F90:406-881.  Call residual(flags | RES_STORE_WALL) first (as the
        reference's getSolution does through blocketteRes(useStoreWall=.true.))."""
        rp = (C.c_double * 3)(*ref_point)
        out = (C.c_double * 12)()
        check(self.L.adfb_forces(level, rp, float(p_ref), out), "adfb_forces")
        return np.array(list(out)).reshape(4, 3)

    def evalFunctions(self, lift_dir, drag_dir, mach_coef, surface_ref=1.0, length_ref=1.0, l_ref=1.0, p_ref=1.0,
                      ref_point=(0.0, 0.0, 0.0)):
        """cl, cd, force and moment coefficients as getCostFunctions forms them
        (src/solver/surfaceIntegrations.F90:43-63, 253-300): fact = 2/(gammaInf MachCoef^2 surfaceRef LRef^2 pRef)."""
        F = self.getForces(ref_point, p_ref)
        fact = 2.0 / (self.prm.gammaInf * mach_coef * mach_coef * surface_ref * l_ref * l_ref * p_ref)
        force, moment = F[0] + F[1], F[2] + F[3]
        cforce = fact * force
        cmoment = (fact / (length_ref * l_ref)) * moment
        return {"fx": force[0], "fy": force[1], "fz": force[2], "cfx": cforce[0], "cfy": cforce[1], "cfz": cforce[2],
                "cl": float(np.dot(cforce, lift_dir)), "cd": float(np.dot(cforce, drag_dir)),
                "clp": float(np.dot(fact * F[0], lift_dir)), "clv": float(np.dot(fact * F[1], lift_dir)),
                "cdp": float(np.dot(fact * F[0], drag_dir)), "cdv": float(np.dot(fact * F[1], drag_dir)),
                "cmx": cmoment[0], "cmy": cmoment[1], "cmz": cmoment[2]}

    def synchronize(self):
        check(self.L.adfb_synchronize(), "adfb_synchronize")

    def launchCount(self):
        return int(self.L.adfb_launch_count())

    def graphCount(self):
        """CUDA graphs cached by the context (-1: graphs are off)"""
        return int(self.L.adfb_graph_count())

    def close(self):
        self.L.adfb_finalize()

    # -- pyADflow-named vector API (device gather kernels + one copy) ---------
    def getStateSize(self):
        return int(self.L.adfb_state_size())

    def getStates(self):
        """pyADflow.getStates (:5174) -> nksolver.getstates (NKSolvers.F90:1378)."""
        out = np.zeros(self.getStateSize())
        check(self.L.adfb_get_states(out.ctypes.data, out.size), "adfb_get_states")
        return out

    def setStates(self, states):
        """pyADflow.setStates (:5181) -> nksolver.setstates (NKSolvers.F90:1452)."""
        states = np.ascontiguousarray(states, dtype=np.float64)
        check(self.L.adfb_set_states(states.ctypes.data, states.size), "adfb_set_states")

    def getResidual(self, res=None, flags=RES_FLOW | RES_TURB | RES_UPDATE_INTERMED):
        """pyADflow.getResidual (:5359) -> nksolver.getres (NKSolvers.F90:1413-1450):
        evaluate the residual, return dw/volRef in AoS order."""
        self.residual(flags)
        if res is None:
            res = np.zeros(self.getStateSize())
        check(self.L.adfb_get_res(res.ctypes.data, res.size), "adfb_get_res")
        return res

    # -- NK matrix-free product (FormFunction_mf / MatMFFD, NKSolvers.F90:437, :167) ----
    def formFunction(self, wvec):
        wvec = np.ascontiguousarray(wvec, dtype=np.float64)
        r = np.zeros_like(wvec)
        check(self.L.adfb_form_function(wvec.ctypes.data, r.ctypes.data, wvec.size), "adfb_form_function")
        return r

    def formFunctionPtr(self, w_ptr, r_ptr, n):
        """FormFunction_mf for host vectors given by address (e.g. page-locked torch tensors: with page-locked vectors and
        blocks without exchange partners the call runs as a slab pipeline -- copy in, kernels and copy out overlap)"""
        check(self.L.adfb_form_function(int(w_ptr), int(r_ptr), int(n)), "adfb_form_function")

    def mffdSetBase(self, U):
        U = np.ascontiguousarray(U, dtype=np.float64)
        check(self.L.adfb_mffd_set_base(U.ctypes.data, U.size), "adfb_mffd_set_base")

    def mffdApply(self, a, h=-1.0, out=None):
        """y = (F(U + h a) - F(U)) / h ; h <= 0 -> Walker-Pernice h computed on the device."""
        a = np.ascontiguousarray(a, dtype=np.float64)
        y = np.zeros_like(a) if out is None else out
        check(self.L.adfb_mffd_apply(a.ctypes.data, y.ctypes.data, a.size, float(h)), "adfb_mffd_apply")
        return y

    def mffdApplyDevice(self, a_ptr, y_ptr, n, h=-1.0):
        """the same product for vectors resident on this GPU (raw device pointers, e.g. torch.Tensor.data_ptr())"""
        check(self.L.adfb_mffd_apply_device(a_ptr, y_ptr, int(n), float(h)), "adfb_mffd_apply_device")

    def mffdLastH(self):
        return float(self.L.adfb_mffd_last_h())
