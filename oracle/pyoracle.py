"""ctypes binding of the CPU oracle (oracle/adflow_oracle.c).

TEST INFRASTRUCTURE ONLY -- imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py; never by the product package.
Parity: pinned bit-exact against the translated reference routines (oracle/adflow_oracle.h).
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))


def build(force=False):
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "adflow_oracle.c")
    stale = (not os.path.exists(so)) or any(
        os.path.getmtime(os.path.join(_HERE, f)) > os.path.getmtime(so)
        for f in ("adflow_oracle.c", "adflow_oracle_smooth.c", "adflow_oracle_sa.c", "adflow_oracle_fluxes.c", "adflow_oracle_mg.c", "adflow_oracle_ank.c", "adflow_oracle.h", "orc_internal.h",
                  "../include/adflow_b200.h")
    )
    if force or stale:
        subprocess.check_call(["make", "-s", "-C", _HERE, "all"])
    assert os.path.exists(src)
    return so


class OrcBlock(C.Structure):
    _fields_ = (
        [(n, C.c_int32) for n in ("nx", "ny", "nz", "nw", "rightHanded", "level")]
        + [(n, C.c_void_p) for n in (
            "w", "p", "rlv", "rev", "x", "si", "sj", "sk", "vol", "volRef", "d2Wall",
            "porI", "porJ", "porK", "iblank", "dw", "fw", "ss", "dss",
            "aa", "radI", "radJ", "radK", "dtl", "grad", "wn", "pn", "scratch", "shock", "wallTau", "wr", "w1", "p1")]
    )


_lib = {}


def lib(fast=False):
    key = "fast" if fast else "strict"
    if key not in _lib:
        build()
        name = "liboracle_fast.so" if fast else "liboracle.so"
        L = C.CDLL(os.path.join(_HERE, name))
        for fn in ("orc_metrics", "orc_volume", "orc_nodal_gradients", "orc_sa_res_scale", "orc_sum_dw_fw"):
            getattr(L, fn).argtypes = [C.c_void_p]
            getattr(L, fn).restype = None
        _lib[key] = L
    return _lib[key]


def orc_block(hb):
    """OrcBlock view of a HostBlock (no copies; arrays must stay alive)."""
    ob = OrcBlock()
    ob.nx, ob.ny, ob.nz, ob.nw = hb.d.nx, hb.d.ny, hb.d.nz, hb.nw
    ob.rightHanded = int(hb.right_handed)
    ob.level = int(getattr(hb, "level", 1))
    for n, _t in OrcBlock._fields_[6:]:
        a = getattr(hb, n)
        assert a.flags.f_contiguous, n
        setattr(ob, n, a.ctypes.data)
    return ob


def _p(x):
    return C.byref(x)


class Oracle:
    """Thin convenience wrapper: Oracle(hb, prm).residual(flags)."""

    def __init__(self, hb, prm, fast=False):
        self.hb, self.prm = hb, prm
        self.L = lib(fast)
        self.ob = orc_block(hb)

    def metrics(self):
        self.L.orc_metrics(_p(self.ob))

    def volume(self):
        self.L.orc_volume(_p(self.ob))

    def pressure(self, include_halos=False):
        self.L.orc_pressure(_p(self.ob), _p(self.prm), C.c_int(int(include_halos)))

    def lam_viscosity(self, include_halos=False):
        self.L.orc_lam_viscosity(_p(self.ob), _p(self.prm), C.c_int(int(include_halos)))

    def eddy_viscosity(self, include_halos=False):
        self.L.orc_eddy_viscosity(_p(self.ob), _p(self.prm), C.c_int(int(include_halos)))

    def residual_core(self, flags, rfil=1.0):
        self.L.orc_residual_core(_p(self.ob), _p(self.prm), C.c_uint(flags), C.c_double(rfil))

    def norms(self):
        out = (C.c_double * 2)()
        self.L.orc_norms(_p(self.ob), _p(self.prm), out)
        return np.array([out[0], out[1]])

    # -- BCs + smoothers (adflow_oracle_smooth.c) ------------------------------
    def _subfaces(self):
        from adflow_b200._lib import AdfbSubface
        subs = self.hb.subfaces
        arr = (AdfbSubface * max(1, len(subs)))()
        self._keep = []
        for q, s in enumerate(subs):
            arr[q].bcType, arr[q].faceId = s["bcType"], s["faceId"]
            arr[q].icBeg, arr[q].icEnd, arr[q].jcBeg, arr[q].jcEnd = s["icBeg"], s["icEnd"], s["jcBeg"], s["jcEnd"]
            arr[q].subsonicInletTreatment = int(s.get("subsonicInletTreatment", 0))
            for name in ("norm", "rface", "uSlip", "TNSWall", "ps", "rho", "velx", "vely", "velz", "ptInlet", "ttInlet", "htInlet",
                         "flowXdirInlet", "flowYdirInlet", "flowZdirInlet", "turbInlet"):
                a = s.get(name)
                if a is not None:
                    a = np.asfortranarray(a, dtype=np.float64)
                    self._keep.append(a)
                    setattr(arr[q], name, a.ctypes.data)
            if s.get("iblank") is not None:   # BCData%iblank, int32 (icBeg:icEnd, jcBeg:jcEnd)
                a = np.asfortranarray(s["iblank"], dtype=np.int32)
                self._keep.append(a)
                arr[q].iblank = a.ctypes.data
        return len(subs), arr

    def apply_turb_bc(self, second_halo=True):
        n, arr = self._subfaces()
        self.L.orc_apply_turb_bc(_p(self.ob), _p(self.prm), C.c_int(n), arr, C.c_int(int(second_halo)))

    def apply_flow_bc(self, second_halo=True):
        n, arr = self._subfaces()
        self.L.orc_apply_flow_bc(_p(self.ob), _p(self.prm), C.c_int(n), arr, C.c_int(int(second_halo)))

    def residual_averaging(self):
        self.L.orc_residual_averaging(_p(self.ob), _p(self.prm))

    def residual_block(self, rfil=1.0):
        self.L.orc_residual_block(_p(self.ob), _p(self.prm), C.c_double(rfil))

    def time_step(self, update_dt=True):
        self.L.orc_time_step(_p(self.ob), _p(self.prm), C.c_int(int(update_dt)))

    def rk_stage(self, stage):
        n, arr = self._subfaces()
        self.L.orc_rk_stage(_p(self.ob), _p(self.prm), C.c_int(stage), C.c_int(n), arr)

    def rk_smoother(self):
        n, arr = self._subfaces()
        self.L.orc_rk_smoother(_p(self.ob), _p(self.prm), C.c_int(n), arr)

    def dadi_step(self):
        n, arr = self._subfaces()
        self.L.orc_dadi_step(_p(self.ob), _p(self.prm), C.c_int(n), arr)

    def compute_dw_dadi(self):
        self.L.orc_compute_dw_dadi(_p(self.ob), _p(self.prm))

    def sa_block(self):
        n, arr = self._subfaces()
        self.L.orc_sa_block(_p(self.ob), _p(self.prm), C.c_int(n), arr)

    def wall_forces(self, ref_point=(0.0, 0.0, 0.0), p_ref=1.0):
        """Fp, Fv, Mp, Mv (each 3) of the wall subfaces; needs a residual evaluation first (stores wallTau)"""
        n, arr = self._subfaces()
        rp = (C.c_double * 3)(*ref_point)
        out = (C.c_double * 12)()
        self.L.orc_wall_forces(_p(self.ob), _p(self.prm), C.c_int(n), arr, rp, C.c_double(p_ref), out)
        return np.array(list(out)).reshape(4, 3)

    def reference_shock_sensor(self):
        self.L.orc_reference_shock_sensor(_p(self.ob), _p(self.prm))

    def call(self, name, *args):
        getattr(self.L, name)(_p(self.ob), *args)

    # -- multigrid (adflow_oracle_mg.c); `self` is the block named first in each docstring -------------------------
    @staticmethod
    def _tab(a, dtype):
        a = np.ascontiguousarray(np.asfortranarray(a, dtype=dtype).ravel(order="F"))
        return a, a.ctypes.data_as(C.c_void_p)

    def residual_block_coarse(self, rfil=1.0, init=1):
        self.L.orc_residual_block_coarse(_p(self.ob), _p(self.prm), C.c_double(rfil), C.c_int(init))

    def diss_scalar_coarse(self, rfil=1.0):
        self.L.orc_diss_scalar_coarse(_p(self.ob), _p(self.prm), C.c_double(rfil))

    def diss_matrix_coarse(self, rfil=1.0):
        self.L.orc_diss_matrix_coarse(_p(self.ob), _p(self.prm), C.c_double(rfil))

    def mg_corner_row_halos(self):
        self.L.orc_mg_corner_row_halos(_p(self.ob), _p(self.prm))

    def mg_restrict(self, fine):
        """COARSE block: restriction of `fine` (an Oracle) into wr / w / p / rev + etot, rlv, rev, corner row halos"""
        mg = self.hb.mg
        keep = [self._tab(mg[n], np.int32) for n in ("mgIFine", "mgJFine", "mgKFine")]
        keep += [self._tab(mg[n], np.float64) for n in ("mgIWeight", "mgJWeight", "mgKWeight")]
        self.L.orc_mg_restrict(_p(self.ob), _p(fine.ob), _p(self.prm), *[k[1] for k in keep])

    def mg_store_w1(self):
        self.L.orc_mg_store_w1(_p(self.ob))

    def mg_forcing(self):
        self.L.orc_mg_forcing(_p(self.ob), _p(self.prm))

    def mg_prolong(self, coarse):
        """FINE block: interpolate the corrections of `coarse` (an Oracle) and update w, p (+ etot, rlv, rev)"""
        mg = self.hb.mg
        keep = [self._tab(mg[n], np.int32) for n in ("mgICoarse", "mgJCoarse", "mgKCoarse")]
        n, arr = coarse._subfaces()
        self.L.orc_mg_prolong(_p(self.ob), _p(coarse.ob), _p(self.prm), C.c_int(n), arr, *[k[1] for k in keep])

    def mg_prolong_solution(self, coarse):
        """FINE block: transferToFineGrid(.false.) -- interpolate the SOLUTION of `coarse` (an Oracle), extrapolate into the halos"""
        mg = self.hb.mg
        keep = [self._tab(mg[n], np.int32) for n in ("mgICoarse", "mgJCoarse", "mgKCoarse")]
        n, arr = coarse._subfaces()
        self.L.orc_mg_prolong_solution(_p(self.ob), _p(coarse.ob), _p(self.prm), C.c_int(n), arr, *[k[1] for k in keep])

    # -- ANK pieces (adflow_oracle_ank.c) ---------------------------------------------------------------------------
    def ank_time_step_block(self, ank, i, j, k):
        n = self.hb.nw if ank.coupled else 5
        out = np.zeros((n, n), order="F")
        self.L.orc_ank_time_step_block(_p(self.ob), _p(self.prm), _p(ank), C.c_int(i), C.c_int(j), C.c_int(k), out.ctypes.data_as(C.c_void_p))
        return out

    def ank_physicality_check(self, ank, w_vec, d_vec, lambda_p):
        """returns the new lambdaP; d_vec is clipped in place (coupled turbulence updates)"""
        n = self.hb.nw if ank.coupled else 5
        f = self.L.orc_ank_physicality_check
        f.restype = C.c_double
        return f(_p(ank), C.c_int(n), C.c_long(w_vec.size // n), w_vec.ctypes.data_as(C.c_void_p), d_vec.ctypes.data_as(C.c_void_p),
                 C.c_double(lambda_p))
