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

import numpy as np

from . import _lib
from ._lib import AdfbSubface, check, ptr

RES_DISS_APPROX, RES_VISC_APPROX, RES_UPDATE_INTERMED = 1, 2, 4
RES_FLOW, RES_TURB, RES_STORE_WALL, RES_SKIP_PREAMBLE = 8, 16, 32, 64


class ADFLOW_B200:
    def __init__(self, prm, device=0, rank=0, nranks=1, unique_id=None):
        self.L = _lib.load()
        check(self.L.adfb_init(device, unique_id, rank, nranks), "adfb_init")
        self.prm = prm
        check(self.L.adfb_set_params(C.byref(prm)), "adfb_set_params")
        self.blocks = []  # HostBlock descriptors (extents only are needed after upload)
        self._keep = []

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
