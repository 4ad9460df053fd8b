"""Parity of the CUDA residual path (through the C ABI) with the CPU oracle.

Tolerance: north_star asks for residuals within 1e-10 relative of the reference;
the oracle and the kernels keep the same per-cell summation order, so the tests
hold the CUDA path to 1e-12 (relative L2 per variable and relative max-norm) --
the slack covers FMA contraction and libm/libdevice pow/exp differences."""
import os

import numpy as np
import pytest

from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_SKIP_PREAMBLE, RES_TURB

from util import case, oracle_residual, rel_l2, rel_max

pytestmark = pytest.mark.gpu

TOL = 1e-12
GENERAL_KERNELS = os.environ.get("ADFB_FUSED") == "0"


def run_cuda(prm, hb, flags, upload_metrics=True):
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb, upload_metrics=upload_metrics)
        s.residual(flags | RES_SKIP_PREAMBLE)
        dw = s.downloadResidual(0)
        inter = s.downloadIntermed(0)
        norms = s.getResNorms()
        extra = {"grad": s.downloadArray(0, "grad", 12), "dss": s.downloadArray(0, "dss", 3),
                 "aa": s.downloadArray(0, "aa")}
    finally:
        s.close()
    return dw, inter, norms, extra


def compare(prm, hb, flags, tol=TOL, upload_metrics=True):
    ref = oracle_residual(prm, hb, flags)
    dw, inter, norms, extra = run_cuda(prm, hb, flags, upload_metrics)
    ow = hb.d.owned()
    nvar = hb.nw if (flags & RES_TURB) else 5
    l0 = 0 if (flags & RES_FLOW) else 5
    for l in range(l0, nvar):
        a, b = dw[ow + (l,)], ref.dw[ow + (l,)]
        assert np.isfinite(a).all()
        assert rel_l2(a, b) < tol, "dw[%d] rel L2 %.3e" % (l, rel_l2(a, b))
        assert rel_max(a, b) < 10 * tol, "dw[%d] rel max %.3e" % (l, rel_max(a, b))
    d = hb.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    for n in ("radI", "radJ", "radK"):
        assert rel_max(inter[n], getattr(ref, n)[c1]) < tol, n
    assert rel_max(inter["dtl"][1:-1, 1:-1, 1:-1], ref.dtl[ow]) < tol
    return ref, dw, norms, extra


@pytest.mark.parametrize("shape", [(16, 12, 8), (33, 9, 7), (5, 6, 40), (1, 1, 1), (2, 35, 3)])
def test_rans_sa_residual_matches_oracle(cuda_lib, shape):
    prm, hb = case(*shape)
    ref, dw, norms, extra = compare(prm, hb, RES_FLOW | RES_TURB)
    from oracle.pyoracle import Oracle
    rn = Oracle(ref, prm).norms()
    assert abs(norms[0] - rn[0]) <= 1e-11 * rn[0]
    assert abs(norms[1] - rn[1]) <= 1e-11 * rn[1]
    d = hb.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    assert rel_max(extra["aa"][c1], ref.aa[c1]) < TOL
    if GENERAL_KERNELS:   # nodal gradients and shock sensor only exist in HBM on the general (k_nodal/k_faces/k_div) path
        nodes = (slice(1, d.il + 1), slice(1, d.jl + 1), slice(1, d.kl + 1))
        assert rel_max(extra["grad"][nodes], ref.grad[nodes]) < TOL
        assert rel_max(extra["dss"][c1], ref.dss[c1]) < 1e-9  # sensor is a ratio of small differences


@pytest.mark.skipif(GENERAL_KERNELS, reason="already the ADFB_FUSED=0 run")
def test_general_kernels_still_match(cuda_lib):
    """The tile kernel (fused_kernels.cuh) is the default for the exact scalar-JST residual; the general kernels it
    replaces there still serve every other option, so the same parity files are re-run with ADFB_FUSED=0."""
    import subprocess
    import sys
    env = dict(os.environ, ADFB_FUSED="0")
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(here, "test_residual_parity.py"), os.path.join(here, "test_cuda_vs_reference.py"),
                        os.path.join(here, "test_smoother_parity.py"), os.path.join(here, "test_regimes_gpu.py"), "-m", "gpu", "-q", "-x"], env=env, capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


def test_flow_only_and_turb_only(cuda_lib):
    prm, hb = case(12, 10, 9)
    compare(prm, hb, RES_FLOW)
    compare(prm, hb, RES_TURB)


@pytest.mark.parametrize("options", [
    {"equationType": "Euler"},
    {"equationType": "laminar NS"},
    {"useQCR": True},
    {"turbulenceOrder": "second order"},
    {"turbulenceProduction": "vorticity"},
    {"useft2SA": False},
    {"vis2": 0.5, "vis4": 1.0 / 64, "dissipationScalingExponent": 2.0 / 3.0},
    {"discretization": "central plus matrix dissipation"},
    {"discretization": "central plus matrix dissipation", "equationType": "Euler"},
    {"discretization": "upwind"},
    {"discretization": "upwind", "limiter": "minmod"},
    {"discretization": "upwind", "limiter": "no limiter", "equationType": "laminar NS"},
    {"discretization": "upwind", "limiter": "first order", "equationType": "Euler"},
])
def test_option_variants(cuda_lib, options):
    prm, hb = case(14, 11, 10, options)
    flags = RES_FLOW | (RES_TURB if prm.equations == 3 else 0)
    compare(prm, hb, flags)


def test_metrics_computed_on_device(cuda_lib):
    """si/sj/sk = NULL -> blockette `metrics` runs on the device."""
    prm, hb = case(10, 9, 8)
    compare(prm, hb, RES_FLOW | RES_TURB, upload_metrics=False)


def test_porosity_and_iblank(cuda_lib):
    prm, hb = case(12, 10, 8)
    d = hb.d
    hb.porI[5, :, :] = -1   # noFlux plane
    hb.porJ[:, 4, :] = 0    # boundFlux plane
    hb.iblank[4:7, 4:6, 3:5] = 0
    hb.iblank[8, 8, 6] = -1
    compare(prm, hb, RES_FLOW | RES_TURB)


def test_free_stream_preservation_on_device(cuda_lib):
    from test_oracle_invariants import freestream_block
    prm, hb = freestream_block(16, 12, 8)
    dw, *_ = run_cuda(prm, hb, RES_FLOW | RES_TURB)
    ow = hb.d.owned()
    scale = np.abs(hb.si[ow]).max() * prm.wInf[1] * prm.wInf[4]
    for l in range(5):
        assert np.abs(dw[ow + (l,)]).max() < 1e-13 * scale


def test_vector_api_roundtrip(cuda_lib):
    """getStates/setStates/getResidual ordering (NKSolvers.F90:1378-1485)."""
    prm, hb = case(7, 6, 5)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        ow = hb.d.owned()
        st = s.getStates()
        exp = np.transpose(hb.w[ow], (2, 1, 0, 3)).reshape(-1)
        assert np.array_equal(st, exp)
        s.setStates(st * 1.0)
        assert np.array_equal(s.getStates(), exp)
        res = s.getResidual(flags=RES_FLOW | RES_TURB | RES_SKIP_PREAMBLE)
        ref = oracle_residual(prm, hb)
        rexp = np.transpose(ref.dw[ow] / hb.volRef[ow][..., None], (2, 1, 0, 3)).reshape(-1)
        assert rel_l2(res, rexp) < TOL
    finally:
        s.close()


def test_state_prep_matches_oracle(cuda_lib):
    """p, rlv, rev on owned cells (blocketteRes preamble :213-218) via adfb_residual without SKIP."""
    from oracle.pyoracle import Oracle
    prm, hb = case(9, 8, 7)
    hb.subfaces = []
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    hb2 = hb.copy()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb2)
        s.residual(RES_FLOW | RES_TURB)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    ow = hb.d.owned()
    assert rel_max(p[ow], ho.p[ow]) < 1e-14
    assert rel_max(rlv[ow], ho.rlv[ow]) < 1e-13
    assert rel_max(rev[ow], ho.rev[ow]) < 1e-12
