"""Option / reference-state handling for the hot path.

Mirrors the part of the reference that turns the Python option dict and the
AeroProblem into the Fortran module globals the flux routines read:

* defaults: ``adflow/pyADflow.py:5632-5940`` (vis2 0.25, vis4 0.0156, CFL 1.7,
  adis 0.67, useft2SA True, turbulenceProduction strain, nSubiterTurb 3 ...)
  layered over ``src/inputParam/inputParamRoutines.F90:3790-4000``;
* non-dimensionalisation: ``referenceState``
  (``src/initFlow/initializeFlow.F90:10-182``);
* Runge-Kutta tables: ``src/inputParam/inputParamRoutines.F90:3576-3633``.

The result is the ``AdfbParams`` POD of ``include/adflow_b200.h``.
"""
import ctypes as C
import math

import numpy as np


class AdfbParams(C.Structure):
    """ctypes twin of ``struct AdfbParams`` (include/adflow_b200.h)."""

    _fields_ = [
        ("gammaInf", C.c_double), ("RGas", C.c_double), ("pInfCorr", C.c_double), ("rhoInf", C.c_double),
        ("wInf", C.c_double * 6), ("pInf", C.c_double),
        ("muSuth", C.c_double), ("TSuth", C.c_double), ("SSuth", C.c_double),
        ("prandtl", C.c_double), ("prandtlTurb", C.c_double),
        ("vis2", C.c_double), ("vis4", C.c_double), ("adis", C.c_double), ("acousticScaleFactor", C.c_double),
        ("kappaCoef", C.c_double),
        ("rsaK", C.c_double), ("rsaCb1", C.c_double), ("rsaCb2", C.c_double), ("rsaCb3", C.c_double),
        ("rsaCv1", C.c_double), ("rsaCw1", C.c_double), ("rsaCw2", C.c_double), ("rsaCw3", C.c_double),
        ("rsaCt3", C.c_double), ("rsaCt4", C.c_double), ("rsaCrot", C.c_double),
        ("cfl", C.c_double), ("cflCoarse", C.c_double),
        ("etaRK", C.c_double * 6), ("cdisRK", C.c_double * 6),
        ("alfaTurb", C.c_double), ("turbResScale", C.c_double),
        ("cflLimit", C.c_double), ("smoop", C.c_double), ("sigma", C.c_double),
        ("vis2Coarse", C.c_double), ("fcoll", C.c_double),
        ("equations", C.c_int32), ("spaceDiscr", C.c_int32), ("nRKStages", C.c_int32), ("turbProd", C.c_int32),
        ("useQCR", C.c_int32), ("useft2SA", C.c_int32), ("useRotationSA", C.c_int32), ("approxSA", C.c_int32),
        ("secondOrdTurb", C.c_int32), ("limiter", C.c_int32), ("resAveraging", C.c_int32),
        ("nSubiterTurb", C.c_int32), ("wallBCConstantPressure", C.c_int32), ("reserved", C.c_int32),
        ("hScalingInlet", C.c_int32), ("outflowLinearExtrapol", C.c_int32),
        ("mgBoundCorr", C.c_int32), ("spaceDiscrCoarse", C.c_int32),
        ("useDissContinuation", C.c_int32), ("pad_", C.c_int32),
        ("dissContMagnitude", C.c_double), ("dissContMidpoint", C.c_double), ("dissContSharpness", C.c_double),
    ]


class AdfbAnkParams(C.Structure):
    """ctypes twin of ``struct AdfbAnkParams`` (include/adflow_b200.h); defaults = pyADflow's ANK options"""

    _fields_ = [("cfl", C.c_double), ("cflLimit", C.c_double), ("turbCFLScale", C.c_double), ("physLSTol", C.c_double),
                ("physLSTolTurb", C.c_double), ("stepMin", C.c_double), ("stepFactor", C.c_double), ("machInf", C.c_double),
                ("coupled", C.c_int32), ("useDissApprox", C.c_int32), ("useFullVisc", C.c_int32), ("charTimeStepType", C.c_int32)]


def make_ank_params(cfl=5.0, coupled=False, char_time_step="None", mach=0.8, **kw):
    """ANKCFL0 5.0, ANKCFLLimit 1e5, ANKTurbCFLScale 1.0, ANKPhysicalLSTol 0.2, ANKPhysicalLSTolTurb 0.99, ANKStepMin
    0.01, ANKStepFactor 1.0, ANKUseApproxSA ... (adflow/pyADflow.py defaults); first-order (approximate) fluxes are the
    ANK default until ANKSecondOrdSwitchTol"""
    a = AdfbAnkParams()
    a.cfl, a.cflLimit, a.turbCFLScale = cfl, kw.get("cflLimit", 1e5), kw.get("turbCFLScale", 1.0)
    a.physLSTol, a.physLSTolTurb = kw.get("physLSTol", 0.2), kw.get("physLSTolTurb", 0.99)
    a.stepMin, a.stepFactor, a.machInf = kw.get("stepMin", 0.01), kw.get("stepFactor", 1.0), mach
    a.coupled = int(coupled)
    a.useDissApprox, a.useFullVisc = int(kw.get("useDissApprox", True)), int(kw.get("useFullVisc", True))
    a.charTimeStepType = {"None": 0, "VLR": 1, "Turkel": 2}[char_time_step]
    return a


EULER, NS, RANS = 1, 2, 3
DISS_SCALAR, DISS_MATRIX, UPWIND = 1, 2, 4
PROD_STRAIN, PROD_VORTICITY = 1, 2

# pyADflow option table defaults relevant to the path (adflow/pyADflow.py:5632-5940)
DEFAULT_OPTIONS = {
    "equationType": "RANS",
    "discretization": "central plus scalar dissipation",
    "vis2": 0.25,
    "vis4": 0.0156,
    "vis2Coarse": 0.5,
    "coarseDiscretization": "central plus scalar dissipation",
    "MGCycle": "sg",
    "dissipationScalingExponent": 0.67,
    "acousticScaleFactor": 1.0,
    "turbulenceOrder": "first order",
    "turbulenceProduction": "strain",
    "useQCR": False,
    "useRotationSA": False,
    "useft2SA": True,
    "eddyVisInfRatio": 0.009,
    "turbResScale": 10000.0,
    "smoother": "DADI",
    "nRKStages": 5,
    "CFL": 1.7,
    "CFLCoarse": 1.0,
    "CFLLimit": 1.5,
    "nSubiterTurb": 3,
    "nSubiter": 1,
    "resAveraging": "alternate",
    "smoothParameter": 1.5,
    "dissipationLumpingParameter": 6.0,
    "useBlockettes": True,
    "liftIndex": 2,
    "viscWallTreatment": "constant pressure extrapolation",
    "useApproxSA": False,
    "limiter": "van Albada",
    "kappaCoef": 1.0 / 3.0,
    "useDissContinuation": False,
    "dissContMagnitude": 1.0,
    "dissContMidpoint": 3.0,
    "dissContSharpness": 3.0,
}


def rk_coefficients(n_stages):
    """etaRK / cdisRK tables, src/inputParam/inputParamRoutines.F90:3576-3633."""
    eta = np.zeros(6)
    cdis = np.zeros(6)
    if n_stages == 1:
        eta[0] = 1.0
        cdis[0] = 1.0
    elif n_stages == 2:
        eta[:2] = [0.2222, 1.0]
        cdis[:2] = [1.0, 1.0]
    elif n_stages == 3:
        eta[:3] = [0.2846, 0.6067, 1.0]
        cdis[:3] = [1.0, 1.0, 1.0]
    elif n_stages == 4:
        eta[:4] = [0.33333333, 0.26666667, 0.55555555, 1.0]
        cdis[:4] = [1.0, 0.5, 0.0, 0.0]
    elif n_stages == 5:
        eta[:5] = [0.25, 0.16666667, 0.37500000, 0.50000000, 1.0]
        cdis[:5] = [1.0, 0.0, 0.56, 0.0, 0.44]
    elif n_stages == 6:
        eta[:6] = [0.0722, 0.1421, 0.2268, 0.3425, 0.5349, 1.0]
        cdis[:6] = [1.0] * 6
    else:
        raise ValueError("nRKStages must be 1..6 (inputParamRoutines.F90:3576)")
    return eta, cdis


def sa_nu_known_eddy_ratio(eddy_ratio, nu_lam, cv1=7.1):
    """saNuKnownEddyRatio, src/turbulence/turbUtils.F90:333-409 (Newton on chi)."""
    if eddy_ratio <= 0.0:
        return 0.0
    cv13 = cv1**3
    if eddy_ratio < 1.0e-4:
        chi = 0.5
    elif eddy_ratio < 1.0:
        chi = 5.0
    elif eddy_ratio < 10.0:
        chi = 10.0
    else:
        chi = eddy_ratio
    while True:
        chi2 = chi * chi
        chi3 = chi * chi2
        chi4 = chi * chi3
        f = chi4 - eddy_ratio * (chi3 + cv13)
        df = 4.0 * chi3 - 3.0 * eddy_ratio * chi2
        dchi = f / df
        chi = chi - dchi
        if abs(dchi / chi) <= 1.0e-10:
            break
    return nu_lam * chi


def make_params(options=None, mach=0.8, alpha_deg=1.8, P=20000.0, T=220.0, R=287.87, gamma=1.4):
    """Build AdfbParams from pyADflow-style options + an AeroProblem.

    AeroProblem defaults are the tutorial wing of the regression tests
    (tests/reg_tests/reg_aeroproblems.py:5-19: M 0.8, alpha 1.8, P 20 kPa, T 220 K).
    Non-dimensionalisation follows referenceState exactly:
    pRef = pInfDim, rhoRef = rhoInfDim, TRef = TInfDim  =>  rhoInf = pInf = 1, RGas = 1.
    """
    opt = dict(DEFAULT_OPTIONS)
    if options:
        unknown = set(options) - set(opt)
        if unknown:
            raise KeyError("unknown option(s): %s" % sorted(unknown))
        opt.update(options)
    prm = AdfbParams()
    eq = {"rans": RANS, "euler": EULER, "laminar ns": NS}[opt["equationType"].lower()]
    prm.equations = eq
    prm.spaceDiscr = {
        "central plus scalar dissipation": DISS_SCALAR,
        "central plus matrix dissipation": DISS_MATRIX,
        "upwind": UPWIND,
    }[opt["discretization"]]
    # Sutherland (inputParamRoutines.F90:4001-4003)
    muSuthDim, TSuthDim, SSuthDim = 1.716e-5, 273.15, 110.55
    rhoInfDim = P / (R * T)
    muInfDim = muSuthDim * ((TSuthDim + SSuthDim) / (T + SSuthDim)) * ((T / TSuthDim) ** 1.5)
    pRef, TRef, rhoRef = P, T, rhoInfDim
    muRef = math.sqrt(pRef * rhoRef)
    pInf = P / pRef
    rhoInf = rhoInfDim / rhoRef
    uInf = mach * math.sqrt(gamma * pInf / rhoInf)
    RGas = R * rhoRef * TRef / pRef
    muInf = muInfDim / muRef
    prm.gammaInf = gamma
    prm.RGas = RGas
    prm.pInf = pInf
    prm.pInfCorr = pInf
    prm.rhoInf = rhoInf
    prm.muSuth = muSuthDim / muRef
    prm.TSuth = TSuthDim / TRef
    prm.SSuth = SSuthDim / TRef
    prm.prandtl = 0.72
    prm.prandtlTurb = 0.90
    # free-stream direction: alpha about the z axis for liftIndex 2 (pyADflow.py:1144 ff.)
    a = math.radians(alpha_deg)
    if opt["liftIndex"] == 2:
        vdir = (math.cos(a), math.sin(a), 0.0)
    else:
        vdir = (math.cos(a), 0.0, math.sin(a))
    w = [rhoInf, uInf * vdir[0], uInf * vdir[1], uInf * vdir[2], 0.0, 0.0]
    # SA constants (adflow/pyADflow.py:5709-5720; src/modules/paramTurb.F90)
    prm.rsaK, prm.rsaCb1, prm.rsaCb2, prm.rsaCb3 = 0.41, 0.1355, 0.622, 0.66666666667
    prm.rsaCv1, prm.rsaCw2, prm.rsaCw3 = 7.1, 0.3, 2.0
    prm.rsaCt3, prm.rsaCt4, prm.rsaCrot = 1.2, 0.5, 2.0
    prm.rsaCw1 = prm.rsaCb1 / (prm.rsaK**2) + (1.0 + prm.rsaCb2) / prm.rsaCb3
    if eq == RANS:
        w[5] = sa_nu_known_eddy_ratio(opt["eddyVisInfRatio"], muInf / rhoInf, prm.rsaCv1)
    # etot (flowUtils.F90:674): rho*(p/((g-1) rho) + 0.5 u^2)
    w[4] = rhoInf * (pInf / ((gamma - 1.0) * rhoInf) + 0.5 * uInf * uInf)
    for i in range(6):
        prm.wInf[i] = w[i]
    prm.vis2, prm.vis4 = opt["vis2"], opt["vis4"]
    # multigrid: vis2Coarse (pyADflow default 0.5), fcoll = 1 and mgBoundCorr = bcDirichlet0 are not pyADflow options
    # (inputParamRoutines.F90:3921-3923)
    prm.vis2Coarse, prm.fcoll, prm.mgBoundCorr = opt["vis2Coarse"], 1.0, 0
    prm.spaceDiscrCoarse = {"central plus scalar dissipation": DISS_SCALAR, "central plus matrix dissipation": DISS_MATRIX,
                            "upwind": UPWIND}[opt["coarseDiscretization"]]
    prm.adis = opt["dissipationScalingExponent"]
    prm.acousticScaleFactor = opt["acousticScaleFactor"]
    prm.kappaCoef = opt["kappaCoef"]
    prm.cfl, prm.cflCoarse = opt["CFL"], opt["CFLCoarse"]
    prm.nRKStages = opt["nRKStages"]
    eta, cdis = rk_coefficients(opt["nRKStages"])
    for i in range(6):
        prm.etaRK[i] = eta[i]
        prm.cdisRK[i] = cdis[i]
    prm.alfaTurb = 0.8
    prm.turbResScale = opt["turbResScale"]
    prm.cflLimit = opt["CFLLimit"]
    prm.smoop = opt["smoothParameter"]
    prm.sigma = opt["dissipationLumpingParameter"]
    prm.turbProd = {"strain": PROD_STRAIN, "vorticity": PROD_VORTICITY}[opt["turbulenceProduction"]]
    prm.useQCR = int(opt["useQCR"])
    prm.useft2SA = int(opt["useft2SA"])
    prm.useRotationSA = int(opt["useRotationSA"])
    prm.approxSA = int(opt["useApproxSA"])
    prm.secondOrdTurb = int(opt["turbulenceOrder"] == "second order")
    prm.limiter = {"first order": 0, "no limiter": 1, "van Albada": 2, "minmod": 3}[opt["limiter"]]
    prm.resAveraging = {"never": 0, "always": 1, "alternate": 2}[opt["resAveraging"]]
    prm.nSubiterTurb = opt["nSubiterTurb"]
    prm.wallBCConstantPressure = int(opt["viscWallTreatment"] == "constant pressure extrapolation")
    prm.useDissContinuation = int(opt["useDissContinuation"])
    prm.dissContMagnitude, prm.dissContMidpoint = opt["dissContMagnitude"], opt["dissContMidpoint"]
    prm.dissContSharpness = opt["dissContSharpness"]
    prm._muInf = muInf  # convenience for the synthetic-state generator (not part of the POD)
    return prm
