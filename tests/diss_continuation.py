"""Dissipation-based continuation (useDissContinuation) for the tests: the coefficients the reference forms and the
parameters that make the oracle compute with them.

The reference replaces vis2 of the scalar dissipation by one of two expressions; matrix dissipation, upwinding and the
coarse-level routines have none:

  inviscidDissFluxScalar (blockette.F90:3114-3123, fluxes.F90:1176-1185)
      fis2 = rFil * (vis2 + mag / (1 + exp(-sharp * (log10(totalR / totalR0) + mid))))
      with -sharp * mid as the argument when totalR == 0 or totalR0 == 0
  inviscidDissFluxScalarApprox (blockette.F90:4434-4439)
      fis2 = vis2 + mag / (1 + exp(-sharp * (log10(totalR / totalR0) + mid)))
      no guard: totalR = 0 gives vis2, totalR = totalR0 = 0 gives NaN

The oracle reads vis2 from its parameters and forms rFil * vis2, so a copy of the parameters whose vis2 is the
coefficient above makes it compute the reference's residual with continuation bit for bit.  exp and log10 are those of
the C math library, which the library's host code and the translated reference call as well."""
import ctypes as C
import ctypes.util

from adflow_b200.params import AdfbParams

_M = C.CDLL(ctypes.util.find_library("m"))
_M.exp.restype = _M.log10.restype = C.c_double
_M.exp.argtypes = _M.log10.argtypes = [C.c_double]

SCALAR = "central plus scalar dissipation"
# pyADflow's defaults except the magnitude of the reference's solver-combination test (test_solver_combos.py:76-85)
OPTIONS = {"useDissContinuation": True, "dissContMagnitude": 0.1, "dissContMidpoint": 3.0, "dissContSharpness": 3.0}
# totalR / totalR0 pairs: far from converged, two levels of convergence, and the zero guard from either side
TOTALS = [(2.5, 2.5), (2.5e-3, 2.5), (2.5e-8, 2.5), (0.0, 2.5), (2.5, 0.0)]


def _sigmoid(prm, arg):
    return prm.dissContMagnitude / (1 + _M.exp(-prm.dissContSharpness * arg))


def coef(prm, total_r, total_r0):
    """vis2 of inviscidDissFluxScalar (the rFil factor is the oracle's)"""
    if not prm.useDissContinuation:
        return prm.vis2
    if total_r == 0.0 or total_r0 == 0.0:
        return prm.vis2 + _sigmoid(prm, prm.dissContMidpoint)
    return prm.vis2 + _sigmoid(prm, _M.log10(total_r / total_r0) + prm.dissContMidpoint)


def coef_approx(prm, total_r, total_r0):
    """vis2 of inviscidDissFluxScalarApprox: no guard"""
    if not prm.useDissContinuation:
        return prm.vis2
    ratio = total_r / total_r0 if total_r0 != 0.0 else (float("nan") if total_r == 0.0 else float("inf"))
    return prm.vis2 + _sigmoid(prm, _M.log10(ratio) + prm.dissContMidpoint)


def oracle_params(prm, total_r, total_r0, approx=False):
    """a copy of prm with which the oracle computes the residual of prm with continuation at these totals"""
    q = AdfbParams.from_buffer_copy(prm)
    q.vis2 = (coef_approx if approx else coef)(prm, total_r, total_r0)
    q.useDissContinuation = 0
    return q


def plain(prm):
    """a copy of prm without continuation"""
    q = AdfbParams.from_buffer_copy(prm)
    q.useDissContinuation = 0
    return q
