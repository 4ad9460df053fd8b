"""Harness around oracle/_ref/libblockette_ref.so -- the reference's OWN blockette routines
(`/root/reference/src/NKSolver/blockette.F90`), machine-translated Fortran -> C by
oracle/f90toc.py and compiled with gcc (oracle/Makefile target `ref`).

Test infrastructure only.  The library exists only where /root/reference was present at build
time (this container); on the GPU box the prebuilt .so travels with the snapshot.  `available()`
says whether it can be used; tests that need it skip otherwise.

The translated routines read the module variables of other reference modules; those are plain
C globals in the library (oracle/ref_env.h) and are set here by symbol name.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_ref", "libblockette_ref.so")
_SO_FAST = os.path.join(_HERE, "_ref", "libblockette_ref_fast.so")

FLAG_DISS_APPROX, FLAG_VISC_APPROX, FLAG_UPDATE_INTERMED, FLAG_FLOW, FLAG_TURB, FLAG_STORE_WALL = 1, 2, 4, 8, 16, 32


def available(fast=False):
    return os.path.exists(_SO_FAST if fast else _SO)


_L = None
_BOUND = None


def use_fast(flag=True):
    """select the -O3 -ffast-math build (timing only; the strict build is the one tests compare with)"""
    global _L
    _L = C.CDLL(os.path.abspath(_SO_FAST if flag else _SO))


def lib():
    global _L
    if _L is None:
        _L = C.CDLL(os.path.abspath(_SO))
    return _L


def _seti(name, v):
    C.c_int.in_dll(lib(), name).value = int(v)


def _setd(name, v):
    C.c_double.in_dll(lib(), name).value = float(v)


def _setp(name, arr):
    C.c_void_p.in_dll(lib(), name).value = arr.ctypes.data


# reference enumerations (src/modules/constants.F90) for the values AdfbParams encodes differently
_REF_SPACEDISCR = {1: 1, 2: 2, 4: 9}            # dissScalar, dissMatrix, upwind
_REF_RESAVG = {0: 0, 1: 1, 2: 2}                # noResAveraging, alwaysResAveraging, alternateResAveraging
_REF_LIMITER = {0: 1, 1: 2, 2: 3, 3: 4}         # firstOrder, noLimiter, vanAlbeda, minmod


def set_params(prm, nw, rfil=1.0):
    """inputPhysics / inputDiscretization / flowVarRefState / paramTurb / iteration from AdfbParams."""
    _seti("nw", nw); _seti("nwf", 5); _seti("nt1", 6); _seti("nt2", nw)
    _seti("viscous", prm.equations != 1); _seti("kpresent", 0); _seti("eddymodel", prm.equations == 3)
    _seti("equations", prm.equations); _seti("equationmode", 1); _seti("turbmodel", 2)
    _seti("turbprod", prm.turbProd); _seti("useqcr", prm.useQCR); _seti("useft2sa", prm.useft2SA)
    _seti("userotationsa", prm.useRotationSA)
    _seti("spacediscr", _REF_SPACEDISCR[prm.spaceDiscr]); _seti("limiter", _REF_LIMITER[prm.limiter])
    _seti("orderturb", 2 if prm.secondOrdTurb else 1); _seti("precond", 1); _seti("riemann", 1)
    _seti("riemanncoarse", 1); _seti("approxsa", prm.approxSA)
    _seti("usedisscontinuation", 0); _seti("currentlevel", 1); _seti("groundlevel", 1)
    _seti("lumpeddiss", 0); _seti("viscpc", 0); _seti("spacediscrcoarse", _REF_SPACEDISCR[prm.spaceDiscr]); _seti("smoother", 1)
    _seti("nrkstages", prm.nRKStages)
    # inputParamRoutines.F90:2824-2833: directional scaling and stored radii only with scalar dissipation
    scalar = int(prm.spaceDiscr == 1)
    _seti("dirscaling", scalar); _seti("radiineededfine", scalar); _seti("radiineededcoarse", scalar)
    _seti("ntimeintervalsspectral", 1); _seti("oversetpresent", 0)
    for n in ("pInfCorr", "rhoInf", "gammaInf", "RGas", "prandtl", "prandtlTurb", "vis2", "vis4", "sigma", "adis",
              "acousticScaleFactor", "kappaCoef", "rsaK", "rsaCb1", "rsaCb2", "rsaCb3", "rsaCv1", "rsaCw1", "rsaCw2",
              "rsaCw3", "rsaCt3", "rsaCt4", "rsaCrot"):
        _setd(n.lower(), getattr(prm, n))
    # cpConstant gas; Sutherland constants are stored non-dimensional in AdfbParams (muRef = Tref = 1)
    _seti("cpmodel", 1); _setd("gammaconstant", prm.gammaInf); _setd("pinf", prm.pInf)
    _setd("musuthdim", prm.muSuth); _setd("tsuthdim", prm.TSuth); _setd("ssuthdim", prm.SSuth); _setd("muref", 1.0)
    # smoothers (inputIteration)
    _setd("cfl", prm.cfl); _setd("cflcoarse", prm.cflCoarse); _setd("cfllimit", prm.cflLimit)
    _setd("smoop", prm.smoop); _seti("resaveraging", _REF_RESAVG[prm.resAveraging]); _seti("bp_ndom", 1)
    _seti("exchangepressureearly", 0); _seti("lowspeedpreconditioner", 0)
    eta = (C.c_double * 6).in_dll(lib(), "etark")
    cdis = (C.c_double * 6).in_dll(lib(), "cdisrk")
    for q in range(6):
        eta[q], cdis[q] = prm.etaRK[q], prm.cdisRK[q]
    _setd("timeref", 1.0); _setd("tref", 1.0); _setd("rfil", rfil); _setd("totalr", 1.0); _setd("totalr0", 1.0)
    # module sa derived constants, src/turbulence/sa.F90:123-126
    _setd("sa_cv13", prm.rsaCv1 ** 3); _setd("sa_kar2inv", 1.0 / (prm.rsaK ** 2))
    _setd("sa_cw36", prm.rsaCw3 ** 6); _setd("sa_cb3inv", 1.0 / prm.rsaCb3)
    _setd("alfaturb", prm.alfaTurb); _seti("turbrelax", 2)  # turbRelaxImplicit
    trs = (C.c_double * 4).in_dll(lib(), "turbresscale")
    trs[0] = prm.turbResScale


def ref_constants():
    """integer `parameter`s of the reference's constants.F90, read from the generated header"""
    import re

    out = {}
    with open(os.path.join(_HERE, "_ref", "ref_constants.h")) as f:
        for line in f:
            m = re.match(r"enum \{ (\w+) = \(?(-?\d+)\)? \};", line)
            if m:
                out[m.group(1)] = int(m.group(2))
    return out


class RefSubface(C.Structure):
    _fields_ = [("icbeg", C.c_int), ("icend", C.c_int), ("jcbeg", C.c_int), ("jcend", C.c_int),
                ("norm", C.c_void_p), ("rface", C.c_void_p), ("uslip", C.c_void_p), ("tns_wall", C.c_void_p),
                ("inbeg", C.c_int), ("inend", C.c_int), ("jnbeg", C.c_int), ("jnend", C.c_int),
                ("iblank", C.c_void_p), ("tau", C.c_void_p)] + [
                    (n, C.c_void_p) for n in ("ps", "rho", "velx", "vely", "velz", "ptinlet", "ttinlet", "htinlet", "flowxdirinlet",
                                              "flowydirinlet", "flowzdirinlet", "turbinlet")] + [
                    ("subsonicinlettreatment", C.c_int), ("pad_", C.c_int)]


# AdfbSubface.bcType (include/adflow_b200.h) -> name of the reference's BC constant
_BC_NAME = {1: "symm", 2: "nswalladiabatic", 3: "farfield", 4: "eulerwall", 5: "extrap", 6: "nswallisothermal",
            7: "subsonicoutflow", 8: "subsonicinflow", 9: "supersonicinflow", 10: "supersonicoutflow", 11: "symmpolar"}


def bind_bcs(hb, prm, other_level=False):
    """nBocos / nViscBocos / BCType / BCFaceID / BCData of blockPointers from hb.subfaces.  The reference
    numbers the viscous wall subfaces first (1..nViscBocos); the relative order is otherwise kept.
    other_level: fill flowDoms(nn, coarseLevel)%{nBocos, BCType, BCFaceID, BCData} (cl_*, cbcd) instead."""
    cst = ref_constants()
    subs = sorted(hb.subfaces, key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    nvisc = sum(1 for s_ in subs if s_["bcType"] in (2, 6)) if prm.equations != 1 else 0
    pre = "cl_" if other_level else "bp_"
    _seti(pre + "nbocos", len(subs))
    if not other_level:
        _seti("bp_nviscbocos", nvisc)
    bct = (C.c_int * 64).in_dll(lib(), pre + "bctype")
    bcf = (C.c_int * 64).in_dll(lib(), pre + "bcfaceid")
    tab = (RefSubface * 64).in_dll(lib(), "cbcd" if other_level else "bcd")
    keep = []
    for q, s_ in enumerate(subs):
        bct[q] = cst[_BC_NAME[s_["bcType"]]]
        bcf[q] = s_["faceId"]
        tab[q].icbeg, tab[q].icend, tab[q].jcbeg, tab[q].jcend = s_["icBeg"], s_["icEnd"], s_["jcBeg"], s_["jcEnd"]
        na, nb = s_["icEnd"] - s_["icBeg"] + 1, s_["jcEnd"] - s_["jcBeg"] + 1
        for field, key, ncomp in (("norm", "norm", 3), ("rface", "rface", 1), ("uslip", "uSlip", 3),
                                  ("tns_wall", "TNSWall", 1)):
            a = s_.get(key)
            a = np.zeros((na, nb, ncomp), order="F") if a is None else np.asfortranarray(a, dtype=np.float64)
            keep.append(a)
            setattr(tab[q], field, a.ctypes.data)
        for field, key in (("ps", "ps"), ("rho", "rho"), ("velx", "velx"), ("vely", "vely"), ("velz", "velz"),
                           ("ptinlet", "ptInlet"), ("ttinlet", "ttInlet"), ("htinlet", "htInlet"),
                           ("flowxdirinlet", "flowXdirInlet"), ("flowydirinlet", "flowYdirInlet"),
                           ("flowzdirinlet", "flowZdirInlet"), ("turbinlet", "turbInlet")):
            a = s_.get(key)
            a = np.zeros((na, nb), order="F") if a is None else np.asfortranarray(a, dtype=np.float64)
            keep.append(a)
            setattr(tab[q], field, a.ctypes.data)
        tab[q].subsonicinlettreatment = int(s_.get("subsonicInletTreatment", 0))
        # node range (owned face cells inBeg+1:inEnd), BCData%iblank and viscSubface%tau planes of the subface
        d = hb.d
        face = s_["faceId"]
        la, lb = {1: (d.jl, d.kl), 2: (d.jl, d.kl), 3: (d.il, d.kl), 4: (d.il, d.kl), 5: (d.il, d.jl), 6: (d.il, d.jl)}[face]
        tab[q].inbeg, tab[q].inend = max(s_["icBeg"], 2) - 1, min(s_["icEnd"], la)
        tab[q].jnbeg, tab[q].jnend = max(s_["jcBeg"], 2) - 1, min(s_["jcEnd"], lb)
        ra, rb = slice(s_["icBeg"], s_["icEnd"] + 1), slice(s_["jcBeg"], s_["jcEnd"] + 1)
        fplane = {1: 1, 2: d.il, 3: 1, 4: d.jl, 5: 1, 6: d.kl}[face]      # index of the boundary face
        ax = (face - 1) // 2

        def plane(arr, idx):
            sl = [ra, rb]
            sl.insert(ax, idx)
            return arr[tuple(sl)]

        # BCData%iblank: the subface's own surface blanking, 1 where the host gives none (BCData.F90:2182)
        ib_ = s_.get("iblank")
        ib_ = np.ones((na, nb), dtype=np.int32, order="F") if ib_ is None else np.asfortranarray(ib_, dtype=np.int32)
        assert ib_.shape == (na, nb), ib_.shape
        keep.append(ib_)
        tab[q].iblank = ib_.ctypes.data
        tau = np.asfortranarray(plane(hb.wallTau, fplane)[..., 9 * ax:9 * ax + 6].astype(np.float64))
        keep.append(tau)
        tab[q].tau = tau.ctypes.data
    _seti("viscwallbctreatment", cst["constantpressure"] if prm.wallBCConstantPressure else cst["linextrapolpressure"])
    _seti("eulerwallbctreatment", cst["constantpressure"] if prm.reserved else cst["linextrapolpressure"])
    _seti("hscalinginlet", prm.hScalingInlet)
    _seti("outflowtreatment", cst["linextrapol"] if prm.outflowLinearExtrapol else cst["constantextrapol"])
    w = (C.c_double * 10).in_dll(lib(), "winf")
    for q in range(6):
        w[q] = prm.wInf[q]
    return keep


class RefBlock:
    """blockPointers view of a HostBlock: every array in the uniform box (0:ib,0:jb,0:kb)."""

    OUT = ["dw", "dtl", "aa", "radi", "radj", "radk", "ux", "uy", "uz", "vx", "vy", "vz", "wx", "wy", "wz", "qx",
           "qy", "qz"]

    def __init__(self, hb, prm, bmt=None):
        d = hb.d
        self.hb = hb
        box = d.box
        self.a = {}
        f = np.asfortranarray
        for ref, mine in (("w", "w"), ("p", "p"), ("rlv", "rlv"), ("rev", "rev"), ("vol", "vol"),
                          ("volref", "volRef"), ("d2wall", "d2Wall"), ("shocksensor", "shock"), ("x", "x"),
                          ("si", "si"), ("sj", "sj"), ("sk", "sk")):
            self.a[ref] = f(getattr(hb, mine).astype(np.float64).copy(order="F"))
        self.a["gamma"] = np.full(box, prm.gammaInf, order="F")
        for n in ("sfacei", "sfacej", "sfacek"):
            self.a[n] = np.zeros(box, order="F")
        self.a["dw"] = f(hb.dw.copy(order="F"))
        self.a["fw"] = f(hb.fw.copy(order="F"))
        self.a["wr"] = f(hb.wr.copy(order="F"))
        self.a["w1"] = f(hb.w1.copy(order="F"))
        self.a["p1"] = f(hb.p1.copy(order="F"))
        # multigrid tables with the reference's declared bounds: mgIFine(1:ie, 2), mgIWeight(2:il), mgICoarse(2:il, 2)
        ext = {"I": (d.ie, d.il), "J": (d.je, d.jl), "K": (d.ke, d.kl)}
        for nm, (e_, l_) in ext.items():
            mg = getattr(hb, "mg", {})
            if "mg%sFine" % nm in mg:
                self.a["mg%sfine" % nm.lower()] = f(np.array(mg["mg%sFine" % nm][1:e_ + 1, :], dtype=np.int32, order="F"))
                self.a["mg%sweight" % nm.lower()] = f(np.array(mg["mg%sWeight" % nm][2:l_ + 1], dtype=np.float64))
            if "mg%sCoarse" % nm in mg:
                self.a["mg%scoarse" % nm.lower()] = f(np.array(mg["mg%sCoarse" % nm][2:l_ + 1, :], dtype=np.int32, order="F"))
        self.a["wn"] = f(hb.wn.copy(order="F"))
        self.a["pn"] = f(hb.pn.copy(order="F"))
        self.a["scratch"] = f(hb.scratch.copy(order="F"))
        self.a["dtl"] = f(hb.dtl.copy(order="F"))
        for n in self.OUT[2:]:
            self.a[n] = np.zeros(box, order="F")
        # spectral radii and speed of sound are INPUTS of the block-path residual (computed by timeStep)
        for ref, mine in (("radi", "radI"), ("radj", "radJ"), ("radk", "radK"), ("aa", "aa")):
            self.a[ref] = f(getattr(hb, mine).copy(order="F"))
        # turbulence BC matrices per block face (block.F90 bmti1(je,ke,nt1:nt2,nt1:nt2) ...); `bmt` is a box
        # array holding the scalar SA value of each boundary face at its first-halo cell
        if bmt is None:
            bmt = np.zeros(box, order="F")
        sl = {"bmti1": bmt[1, 1:d.je + 1, 1:d.ke + 1], "bmti2": bmt[d.ie, 1:d.je + 1, 1:d.ke + 1],
              "bmtj1": bmt[1:d.ie + 1, 1, 1:d.ke + 1], "bmtj2": bmt[1:d.ie + 1, d.je, 1:d.ke + 1],
              "bmtk1": bmt[1:d.ie + 1, 1:d.je + 1, 1], "bmtk2": bmt[1:d.ie + 1, 1:d.je + 1, d.ke]}
        for n, v in sl.items():
            self.a[n] = f(np.array(v, dtype=np.float64, order="F"))
            self.a[n.replace("bmt", "bvt")] = np.zeros(v.shape, order="F")
        self.a["s"] = np.zeros(box + (3,), order="F")
        self.a["globalcell"] = np.zeros(box, dtype=np.int32, order="F")
        self.a["iblank"] = f(hb.iblank.astype(np.int32).copy(order="F"))
        for ref, mine in (("pori", "porI"), ("porj", "porJ"), ("pork", "porK")):
            self.a[ref] = f(getattr(hb, mine).astype(np.int32).copy(order="F"))

    SHARED = ("dw", "fw", "scratch", "wn", "pn", "dtl", "radi", "radj", "radk", "gamma", "rlv")

    def bind(self, shared_from=None):
        """blockPointers <- this block.  shared_from: the finest-level RefBlock whose dw, fw, scratch, wn, pn, dtl,
        radI/J/K, gamma, rlv every level points at (setPointers, utils.F90:3419-3477); default: this block's own."""
        d = self.hb.d
        sh = (shared_from or self).hb.d
        _seti("sh_ib", sh.ib); _seti("sh_jb", sh.jb); _seti("sh_kb", sh.kb)
        for n, v in (("nx", d.nx), ("ny", d.ny), ("nz", d.nz), ("il", d.il), ("jl", d.jl), ("kl", d.kl),
                     ("ie", d.ie), ("je", d.je), ("ke", d.ke), ("ib", d.ib), ("jb", d.jb), ("kb", d.kb)):
            _seti("bp_" + n, v)
        _seti("bp_addgridvelocities", 0); _seti("bp_righthanded", int(self.hb.right_handed))
        _seti("bp_sectionid", 1); _seti("bp_blockismoving", 0); _seti("bp_nbkglobal", 1)
        for n, arr in self.a.items():
            assert arr.flags.f_contiguous
            if shared_from is not None and n in self.SHARED:
                arr = shared_from.a[n]
            _setp("bp_" + n, arr)


def residual_core(hb, prm, flags=FLAG_FLOW | FLAG_TURB, rfil=1.0):
    """blocketteResCore (src/NKSolver/blockette.F90:299-753) on one block; returns the RefBlock
    whose arrays hold dw (and, with FLAG_UPDATE_INTERMED, dtl/rad*/aa/nodal gradients)."""
    set_params(prm, hb.nw, rfil)
    global _BOUND
    rb = RefBlock(hb, prm)
    rb.bind()
    _BOUND = rb  # the library holds raw pointers into rb's arrays: keep them alive for call_core()
    args = [C.byref(C.c_int(1 if flags & m else 0)) for m in
            (FLAG_DISS_APPROX, FLAG_VISC_APPROX, FLAG_UPDATE_INTERMED, FLAG_FLOW, FLAG_TURB, FLAG_STORE_WALL)]
    lib().blocketterescore(*args)
    return rb


def call(hb, prm, routine, *int_args, rkstage=1, rfil=1.0, bmt=None):
    """bind `hb` as the current block (blockPointers) and call one translated reference procedure
    whose dummies are all integer/logical by reference, e.g.
    call(hb, prm, "smoothers_executerkstage", rkstage=3) or
    call(hb, prm, "flowutils_computelamviscosity", 1).  Returns the RefBlock (arrays in .a)."""
    global _BOUND
    set_params(prm, hb.nw, rfil)
    _seti("rkstage", rkstage)
    rb = RefBlock(hb, prm, bmt)
    rb.bind()
    rb.keep = bind_bcs(hb, prm)
    _BOUND = rb
    getattr(lib(), routine)(*[C.byref(C.c_int(int(v))) for v in int_args])
    return rb


def again(routine, *int_args):
    """call another translated procedure on the block bound by the last call()/residual_core()"""
    getattr(lib(), routine)(*[C.byref(C.c_int(int(v))) for v in int_args])
    return _BOUND


def wall_forces(hb, prm, ref_point=(0.0, 0.0, 0.0), p_ref=1.0):
    """wallIntegrationFace (src/solver/surfaceIntegrations.F90:406-881) over every wall subface of hb, after
    setBCPointers(mm, .true.); hb.wallTau must hold the stored wall stresses (viscSubface%tau).  Returns
    Fp, Fv, Mp, Mv as a (4, 3) array (localValues(iFp:), (iFv:), (iMp:), (iMv:))."""
    global _BOUND
    cst = ref_constants()
    set_params(prm, hb.nw)
    _setd("pref", p_ref); _setd("lref", 1.0); _setd("machcoef", 1.0)
    pr = (C.c_double * 3).in_dll(lib(), "pointref")
    for q in range(3):
        pr[q] = ref_point[q]
    rb = RefBlock(hb, prm)
    rb.bind()
    rb.keep = bind_bcs(hb, prm)
    _BOUND = rb
    subs = sorted(hb.subfaces, key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    local = (C.c_double * cst["nlocalvalues"])()
    for mm, s_ in enumerate(subs, start=1):
        if s_["bcType"] in (2, 4, 6):
            lib().setbcpointers(C.byref(C.c_int(mm)), C.byref(C.c_int(1)))
            lib().surfaceintegrations_wallintegrationface(local, C.byref(C.c_int(mm)))
    v = np.array(list(local))
    return np.stack([v[cst[k] - 1:cst[k] + 2] for k in ("ifp", "ifv", "imp", "imv")])


def orphan_average(hb, prm, orphans, w_start, w_end, calc_p, calc_lam, calc_eddy, mu_inf, eddy_ratio):
    """orphanAverage (src/utils/haloExchange.F90:201-354) of the translated reference on block hb; orphans = (n, 3) ints"""
    global _BOUND
    set_params(prm, hb.nw)
    rb = RefBlock(hb, prm)
    rb.bind()
    orph = np.ascontiguousarray(np.asarray(orphans, dtype=np.int32).reshape(-1, 3))
    rb.keep = orph
    _BOUND = rb
    _seti("bp_norphans", len(orph))
    _setp("bp_orphans", orph)
    _setd("muinf", mu_inf); _setd("eddyvisinfratio", eddy_ratio)
    winf = (C.c_double * 10).in_dll(lib(), "winf")   # flowVarRefState wInf(1:nw)
    for q in range(6):
        winf[q] = prm.wInf[q]
    lib().haloexchange_orphanaverage(*[C.byref(C.c_int(int(v))) for v in (w_start, w_end, calc_p, 0, calc_lam, calc_eddy)])
    return rb


def set_int(name, value):
    """set an integer module variable of the translated reference (e.g. "rkstage") between calls"""
    _seti(name, value)


def call_core(flags=FLAG_FLOW | FLAG_TURB):
    """re-run blocketteResCore on the block bound by the last residual_core() (timing loops)"""
    args = [C.byref(C.c_int(1 if flags & m else 0)) for m in
            (FLAG_DISS_APPROX, FLAG_VISC_APPROX, FLAG_UPDATE_INTERMED, FLAG_FLOW, FLAG_TURB, FLAG_STORE_WALL)]
    lib().blocketterescore(*args)


class RefMG:
    """Two grid levels of one block for the translated multigrid routines (src/solver/multiGrid.F90).  setPointers
    (nn, level, sps) of the reference is served by a callback that rebinds blockPointers (bp_*) and BCData (bcd) to
    the block of `level`; the OTHER level's arrays that the transfer routines reach through flowDoms(nn, level, sps)
    are bound once (fl_* = fine block, cl_* / cbcd = coarse block)."""

    def __init__(self, fine_hb, coarse_hb, prm, more_levels=()):
        """fine_hb / coarse_hb: levels 1 and 2; more_levels: HostBlocks of levels 3, 4, ... (executeMGCycle)"""
        global _BOUND
        self.prm = prm
        set_params(prm, fine_hb.nw)
        _setd("vis2coarse", prm.vis2Coarse); _setd("fcoll", prm.fcoll); _seti("mgboundcorr", prm.mgBoundCorr)
        _seti("spacediscrcoarse", _REF_SPACEDISCR[prm.spaceDiscrCoarse])
        _seti("radiineededcoarse", int(prm.spaceDiscrCoarse == 1))   # inputParamRoutines.F90:2824-2833
        _seti("nsubiterturb", prm.nSubiterTurb)
        hbs = [fine_hb, coarse_hb] + list(more_levels)
        self.lv = {q + 1: RefBlock(hb, prm) for q, hb in enumerate(hbs)}
        self.keep = {}
        L = lib()

        def hook(level):
            rb = self.lv[level]
            rb.bind(shared_from=self.lv[1] if level != 1 else None)
            self.keep[level] = bind_bcs(rb.hb, prm)
            # the other levels the transfer routines reach through flowDoms(nn, fineLevel / coarseLevel, sps)
            if level - 1 in self.lv:
                f = self.lv[level - 1]
                for n, v in (("ib", f.hb.d.ib), ("jb", f.hb.d.jb), ("kb", f.hb.d.kb)):
                    _seti("fl_" + n, v)
                for n in ("w", "p", "vol", "rev", "w1", "p1", "iblank"):
                    _setp("fl_" + n, f.a[n])
            if level + 1 in self.lv:
                c = self.lv[level + 1]
                for n in ("il", "jl", "kl", "ie", "je", "ke", "ib", "jb", "kb"):
                    _seti("cl_" + n, getattr(c.hb.d, n))
                for n in ("w", "p", "vol", "rev", "w1", "p1", "iblank"):
                    _setp("cl_" + n, c.a[n])
                self.keep["cl"] = bind_bcs(c.hb, prm, other_level=True)

        self._hook = C.CFUNCTYPE(None, C.c_int)(hook)
        C.c_void_p.in_dll(L, "setpointers_hook").value = C.cast(self._hook, C.c_void_p).value
        hook(2)      # the two-level tests call single routines right away: level 2 bound, fl_ = level 1
        hook(1)      # ... and cl_ = level 2
        _BOUND = self

    def execute_mg_cycle(self, cycling, smoother="RK", n_subiterations=1):
        """executeMGCycle (multiGrid.F90:825-955) on ground level 1 with iteration%cycling = cycling"""
        cyc = (C.c_int * 256).in_dll(lib(), "cycling")
        for q, v in enumerate(cycling):
            cyc[q] = int(v)
        _seti("nstepscycling", len(cycling)); _seti("groundlevel", 1); _seti("currentlevel", 1); _seti("rkstage", 0)
        _seti("smoother", 1 if smoother == "RK" else 2); _seti("nsubiterations", n_subiterations)
        try:
            lib().multigrid_executemgcycle()
        finally:
            _seti("smoother", 1); _seti("nsubiterations", 1)

    def seed_coarse_shared(self):
        """put the coarse block's dw, fw, dtl, radI/J/K, rlv, ... where the reference keeps them: in the finest
        level's arrays at the coarse indices (for tests that start in the middle of a cycle)"""
        dc = self.lv[2].hb.d
        sl = (slice(0, dc.ib + 1), slice(0, dc.jb + 1), slice(0, dc.kb + 1))
        for n in RefBlock.SHARED:
            self.lv[1].a[n][sl] = self.lv[2].a[n]

    def close(self):
        C.c_void_p.in_dll(lib(), "setpointers_hook").value = None
        _seti("currentlevel", 1)

    def call(self, level, routine, *int_args, rkstage=None, ground=1):
        """setPointers(1, level, 1), currentLevel = level (ground level `ground`), then one translated procedure"""
        _seti("currentlevel", level); _seti("groundlevel", ground)
        if rkstage is not None:
            _seti("rkstage", rkstage)
        self._hook(level)
        try:
            getattr(lib(), routine)(*[C.byref(C.c_int(int(v))) for v in int_args])
        finally:
            _seti("groundlevel", 1)
        return self.lv[level]

    def transfer_to_coarse(self):
        """transferToCoarseGrid from level 1: fine residual, restriction, coarse BCs, coarse residual, forcing term"""
        _seti("currentlevel", 1); _seti("groundlevel", 1)
        lib().multigrid_transfertocoarsegrid()
        assert C.c_int.in_dll(lib(), "currentlevel").value == 2

    def transfer_to_fine(self, corrections=True):
        """currentLevel = 1; transferToFineGrid(.true.), or with corrections = False the full-multigrid start-up step
        (ground level 2 -> currentLevel 1 < groundLevel: solution interpolated, halos extrapolated, BCs with second halos)"""
        _seti("currentlevel", 1); _seti("groundlevel", 1 if corrections else 2)
        try:
            lib().multigrid_transfertofinegrid(C.byref(C.c_int(1 if corrections else 0)))
        finally:
            _seti("groundlevel", 1)
