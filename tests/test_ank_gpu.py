"""ANK pieces on the device (adfb_ank_*): the matrix-free operator F(v) = R_approx(v) + timeStepMat v of ANKSolver's
FormFunction_mf, its finite-difference product, and the physicality check -- against the oracle, whose
computeTimeStepBlock / physicalityCheckANK are pinned bit for bit against the reference
(tests/test_oracle_vs_reference_ank.py)."""
import ctypes as C

import numpy as np
import pytest

from adflow_b200.params import make_ank_params
from adflow_b200.solver import ADFLOW_B200, RES_DISS_APPROX, RES_FLOW, RES_TURB, RES_VISC_APPROX
from oracle.pyoracle import Oracle

from util import case, rel_l2

pytestmark = pytest.mark.gpu


def vec_of(hb, ns):
    return np.ascontiguousarray(np.transpose(hb.w[hb.d.owned()][..., :ns], (2, 1, 0, 3)).reshape(-1))


def oracle_blocks(prm, ank, hb):
    """timeStepMat of the state in hb (dtl current): (ncells, ns, ns), cell-major like the vectors"""
    d = hb.d
    o = Oracle(hb, prm)
    out = []
    for k in range(2, d.kl + 1):
        for j in range(2, d.jl + 1):
            for i in range(2, d.il + 1):
                out.append(o.ank_time_step_block(ank, i, j, k))
    return np.array(out)


def oracle_ank_function(prm, ank, hb, T, vec):
    """FormFunction_mf of ANKSolver: setWANK, blocketteRes(approx flags), setRVec(ANK), + timeStepMat * vec"""
    d = hb.d
    ns = hb.nw if ank.coupled else 5
    ow = d.owned()
    h2 = hb.copy()
    h2.w[ow + (slice(0, ns),)] = np.asarray(vec).reshape(d.nz, d.ny, d.nx, ns).transpose(2, 1, 0, 3)
    o = Oracle(h2, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    flags = RES_FLOW | (RES_TURB if ank.coupled else 0)
    if ank.useDissApprox:
        flags |= RES_DISS_APPROX
    if ank.useDissApprox and not ank.useFullVisc:
        flags |= RES_VISC_APPROX
    o.residual_core(flags)
    r = h2.dw[ow][..., :ns] / h2.volRef[ow][..., None]
    if ns > 5:
        r[..., 5] *= prm.turbResScale
    r = np.transpose(r, (2, 1, 0, 3)).reshape(-1, ns)
    v = np.asarray(vec).reshape(-1, ns)
    return (r + np.einsum("qlm,qm->ql", T, v)).reshape(-1)


@pytest.mark.parametrize("options,coupled,kind,fullvisc", [(None, False, "None", True), (None, True, "None", False),
                                                          (None, False, "VLR", True), ({"equationType": "Euler"}, False, "Turkel", True),
                                                          (None, True, "VLR", True), (None, True, "Turkel", False)])
def test_ank_operator_and_product(cuda_lib, options, coupled, kind, fullvisc):
    prm, hb = case(11, 9, 8, options)
    ank = make_ank_params(cfl=5.0, coupled=coupled, char_time_step=kind, mach=0.8, cflLimit=50.0, turbCFLScale=2.0, useFullVisc=fullvisc)
    ns = hb.nw if coupled else 5
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    o.call("orc_speed_of_sound", C.byref(prm))
    o.reference_shock_sensor()
    T = oracle_blocks(prm, ank, hb)
    U = vec_of(hb, ns)
    rng = np.random.default_rng(5)
    v = U * (1.0 + 0.01 * rng.standard_normal(U.size))
    a = rng.standard_normal(U.size) * np.abs(U).clip(1e-6)
    Fref = oracle_ank_function(prm, ank, hb, T, v)
    h = 1e-6
    F0 = oracle_ank_function(prm, ank, hb, T, U)
    yref = (oracle_ank_function(prm, ank, hb, T, U + h * a) - F0) / h
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        s.referenceShockSensor()
        s.residual(RES_FLOW | RES_TURB | 4)        # useUpdateIntermed: dtl, spectral radii (and aa) of the current state
        s.ankTimeStepMat()
        F = s.ankFormFunction(v)
        s.ankMffdSetBase(U)
        y = s.ankMffdApply(a, h)
        y2 = s.ankMffdApply(a, -1.0)
        import torch
        da = torch.from_numpy(a.copy()).cuda()
        dy = torch.zeros_like(da)
        s.ankMffdApplyDevice(da.data_ptr(), dy.data_ptr(), da.numel(), h)
        assert np.array_equal(dy.cpu().numpy(), y)
    finally:
        s.close()
    assert rel_l2(F, Fref) < 1e-11, rel_l2(F, Fref)
    assert rel_l2(y, yref) < 1e-5, rel_l2(y, yref)
    assert rel_l2(y2, yref) < 5e-2     # PETSc's default h: consistent first-order quotient
    # the time-step term is really there: F differs from the bare residual by T v
    assert np.abs(np.einsum("qlm,qm->ql", T, v.reshape(-1, ns))).max() > 0


@pytest.mark.parametrize("coupled", [False, True])
def test_ank_physicality_check(cuda_lib, coupled):
    prm, hb = case(10, 9, 7)
    ank = make_ank_params(coupled=coupled)
    ns = hb.nw if coupled else 5
    wv = vec_of(hb, ns)
    rng = np.random.default_rng(11)
    dv = rng.standard_normal(wv.size) * np.abs(wv) * 0.4
    if coupled:
        dv[5::6][:50] = wv[5::6][:50] * 500.0
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        for lam0 in (1.0, 0.03):
            d_ref = dv.copy()
            lam_ref = Oracle(hb, prm).ank_physicality_check(ank, wv, d_ref, lam0)
            lam, d_dev = s.ankPhysicalityCheck(wv, dv, lam0)
            assert lam == lam_ref and 0 < lam <= lam0
            assert np.array_equal(d_dev, d_ref)
    finally:
        s.close()


def _host_gmres(apply, b, restart, max_its, rtol):
    """reference implementation: right-preconditioned (identity) GMRES(restart), classical Gram-Schmidt, x0 = 0"""
    n = b.size
    x = np.zeros(n)
    bnorm = np.linalg.norm(b)
    its = 0
    r = b.copy()
    rnorm = bnorm
    while its < max_its and rnorm > rtol * bnorm:
        V = np.zeros((restart + 1, n)); H = np.zeros((restart + 1, restart))
        V[0] = r / rnorm
        g = np.zeros(restart + 1); g[0] = rnorm
        k = 0
        for j in range(restart):
            w = apply(V[j])
            h = V[:j + 1] @ w
            w = w - h @ V[:j + 1]
            H[:j + 1, j] = h
            H[j + 1, j] = np.linalg.norm(w)
            V[j + 1] = w / H[j + 1, j]
            its += 1; k = j + 1
            y, *_ = np.linalg.lstsq(H[:k + 1, :k], g[:k + 1], rcond=None)
            rnorm = np.linalg.norm(g[:k + 1] - H[:k + 1, :k] @ y)
            if rnorm <= rtol * bnorm or its >= max_its:
                break
        x = x + y @ V[:k]
        r = b - apply(x)
        rnorm = np.linalg.norm(r)
    return x, its


@pytest.mark.parametrize("kind,coupled,shape", [("None", False, (9, 8, 7)), ("VLR", True, (9, 8, 7)),
                                               ("VLR", True, (40, 32, 16))],   # n = 122 880: the 256 CTAs of the dot products loop
                         ids=["None-False", "VLR-True", "VLR-True-large"])
def test_device_gmres_on_a_linear_operator(cuda_lib, kind, coupled, shape):
    """adfb_gmres_solve on the block-diagonal time-step matrix (a LINEAR operator whose blocks the oracle provides):
    two restart cycles reproduce a host GMRES with the same parameters and the estimate of the recurrence is the true
    residual; with the exact inverse as right preconditioner (a callback on the device vectors) it converges at once"""
    prm, hb = case(*shape)
    ank = make_ank_params(cfl=3.0, coupled=coupled, char_time_step=kind, cflLimit=20.0, turbCFLScale=2.0)
    ns = hb.nw if coupled else 5
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    o.call("orc_speed_of_sound", C.byref(prm))
    T = oracle_blocks(prm, ank, hb)
    apply = lambda v: np.einsum("qlm,qm->ql", T, v.reshape(-1, ns)).reshape(-1)  # noqa: E731
    b = np.random.default_rng(2).standard_normal(T.shape[0] * ns)
    rtol, restart, max_its = 1e-12, 12, 24      # the operator is ill conditioned: 2 cycles of 12, no convergence expected
    import torch

    class DevVec:   # a device pointer as a CUDA array for torch
        def __init__(self, ptr, n, readonly):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, readonly), "version": 2}

    Tinv = torch.linalg.inv(torch.from_numpy(T).cuda())
    calls = []

    def pc(ctx, in_ptr, out_ptr, n):
        v = torch.as_tensor(DevVec(in_ptr, n, False), device="cuda").reshape(-1, ns)   # torch rejects read-only views
        out = torch.as_tensor(DevVec(out_ptr, n, False), device="cuda").reshape(-1, ns)
        out.copy_(torch.einsum("qlm,qm->ql", Tinv, v))
        torch.cuda.synchronize()
        calls.append(n)
        return 0

    PCFN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong)
    pc_c = PCFN(pc)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        s.residual(RES_FLOW | RES_TURB | 4)
        s.ankTimeStepMat()
        x, its, rn = s.gmresSolve(b, op="TSMAT", restart=restart, max_its=max_its, rtol=rtol)
        # right preconditioner = the exact inverse (block-diagonal, applied by torch on the device vectors): A M^-1 = I
        xp = np.zeros_like(b)
        itp, rnp = C.c_int(0), C.c_double(0.0)
        rc = s.L.adfb_gmres_solve(2, b.ctypes.data, xp.ctypes.data, b.size, restart, max_its, 1e-10, 1e-50, C.cast(pc_c, C.c_void_p), None,
                                  C.byref(itp), C.byref(rnp))
        from adflow_b200._lib import check
        check(rc, "adfb_gmres_solve with a preconditioner callback")
    finally:
        s.close()
    xh, its_h = _host_gmres(apply, b, restart, max_its, rtol)
    res = np.linalg.norm(b - apply(x)) / np.linalg.norm(b)
    assert its == its_h == max_its
    assert abs(rn / np.linalg.norm(b) - res) < 1e-6 * res + 1e-12    # the recurrence's estimate is the true residual
    assert res < 1.0
    assert np.linalg.norm(x - xh) < 1e-7 * np.linalg.norm(xh), np.linalg.norm(x - xh) / np.linalg.norm(xh)
    assert itp.value <= 2 and len(calls) >= 2
    assert np.linalg.norm(b - apply(xp)) < 1e-8 * np.linalg.norm(b)


@pytest.mark.parametrize("op", ["ANK", "NK"])
def test_device_gmres_on_the_matrix_free_operators(cuda_lib, op):
    """the finite-difference operators are only approximately linear (the differencing parameter follows ||v||), so the
    check is agreement with a host GMRES that applies the SAME device operator vector by vector"""
    prm, hb = case(10, 8, 7)
    ank = make_ank_params(cfl=2.0, coupled=False)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        if op == "ANK":
            s.ankSetParams(ank)
            s.referenceShockSensor()
            s.residual(RES_FLOW | RES_TURB | 4)
            s.ankTimeStepMat()
            U = vec_of(hb, 5)
            s.ankMffdSetBase(U)
            apply = lambda v: s.ankMffdApply(v, -1.0)  # noqa: E731
        else:
            U = s.getStates()
            s.mffdSetBase(U)
            apply = lambda v: s.mffdApply(v, -1.0)  # noqa: E731
        rtol, restart, max_its = 1e-3, 10, 10
        b = apply(np.random.default_rng(3).standard_normal(U.size) * np.abs(U).clip(1e-6) * 1e-3)   # a right-hand side in the range
        x, its, rn = s.gmresSolve(b, op=op, restart=restart, max_its=max_its, rtol=rtol)
        xh, its_h = _host_gmres(apply, b, restart, max_its, rtol)
    finally:
        s.close()
    assert np.isfinite(x).all() and its >= 1 and abs(its - its_h) <= 1
    assert rn <= np.linalg.norm(b) * (1 + 1e-12)
    assert np.linalg.norm(x - xh) < 2e-2 * np.linalg.norm(xh), np.linalg.norm(x - xh) / np.linalg.norm(xh)


def test_turbulence_ksp_pieces(cuda_lib):
    """decoupled ANK, turbulence KSP: FormFunction_mf_turb (NKSolvers.F90:2540-2612), the matrix-free product over it and
    physicalityCheckANKTurb (:3212-3335) against the oracle (whose check is pinned bit for bit against the reference)."""
    import ctypes as C

    from util import FLOW, TURB, case, rel_l2

    prm, hb = case(12, 9, 8)
    ank = make_ank_params(cfl=5.0, coupled=False, physLSTolTurb=0.99, stepMin=0.01, stepFactor=1.0)
    ow = hb.d.owned()
    U = np.ascontiguousarray(np.transpose(hb.w[ow][..., 5], (2, 1, 0)).reshape(-1))
    rng = np.random.default_rng(5)
    vin = U * (1.0 + 0.01 * rng.standard_normal(U.size))

    def oracle_F(v):
        h2 = hb.copy()
        o = Oracle(h2, prm)
        o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        o.time_step(True)                      # dtl of the last time-step evaluation (state of hb)
        dtl = h2.dtl.copy()
        h2.w[ow + (5,)] = np.transpose(v.reshape(hb.d.nz, hb.d.ny, hb.d.nx), (2, 1, 0))
        o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, hb.d.il, 2, hb.d.jl, 2, hb.d.kl)
        o.residual_core(TURB)
        h2.dtl[...] = dtl
        r = np.empty_like(v)
        o.L.orc_ank_turb_rvec(C.byref(o.ob), C.byref(prm), C.byref(ank), v.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p))
        return r

    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        s.residual(FLOW | TURB | 4)            # refreshes dtl like the residual evaluation before the ANK step
        r = s.ankFormFunctionTurb(vin)
        want = oracle_F(vin)
        assert rel_l2(r, want) < 1e-11, rel_l2(r, want)
        # matrix-free product = difference quotient of two function evaluations
        a = rng.standard_normal(U.size) * np.abs(U)
        h = 1e-6
        s.ankMffdTurbSetBase(U)
        y = s.ankMffdTurbApply(a, h)
        yref = (oracle_F(U + h * a) - oracle_F(U)) / h
        assert rel_l2(y, yref) < 1e-6, rel_l2(y, yref)
        # physicality check
        dv = rng.standard_normal(U.size) * np.abs(U) * 0.4
        dv[:30] = U[:30] * 500.0
        lam, dclip = s.ankPhysicalityCheckTurb(U, dv, 1.0)
        f = Oracle(hb, prm).L.orc_ank_physicality_check_turb
        f.restype = C.c_double
        dref = dv.copy()
        lref = f(C.byref(ank), C.c_long(U.size), U.ctypes.data_as(C.c_void_p), dref.ctypes.data_as(C.c_void_p), C.c_double(1.0))
        assert lam == lref and np.array_equal(dclip, dref) and np.abs(dref - dv).max() > 0
        with pytest.raises(Exception):
            s.ankMffdTurbApply(a[:-1], h)
    finally:
        s.close()
