"""Every device path that reads the cell iblank or the face porosities, against the oracle, on the overset layout of
tests/util.py (overset_layout: a hole inside a two-cell fringe shell, a two-cell fringe slab along jMax, holes in the
first cell layer of the kMin wall, noFlux and boundFlux planes in i, j and k), placed on the seams where kernels go
wrong: the tile and k-chunk seams of a forced ADFB_TILE and ADFB_SA_TILE, the slabs of the form-function pipeline, the
32-line groups of the tiled DADI i sweep and the 8-lane partitions of the SA line solve.  Wall forces are weighted by
the surface iblank BCData%iblank (tests/util.py: blank_wall_surfaces).

Tolerances are those of the existing tests of each entry point.  Every test also runs the oracle without the blanking
and porosities and asserts that they move the compared quantity by more than 1e3 times its tolerance."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from adflow_b200 import make_params
from adflow_b200 import synthetic as syn
from adflow_b200.params import make_ank_params
from adflow_b200.solver import ADFLOW_B200, RES_DISS_APPROX, RES_FLOW, RES_SKIP_PREAMBLE, RES_STORE_WALL, RES_TURB, RES_VISC_APPROX
from oracle import refblockette as rb
from oracle.pyoracle import Oracle

from test_ank_gpu import oracle_ank_function, oracle_blocks, vec_of
from test_sa_tile_gpu import _env
from util import (MIXED, blank_wall_surfaces, case, oracle_form_function, oracle_residual, overset_layout, rel_l2, rel_max,
                  split_faces, wall_layer)

pytestmark = pytest.mark.gpu

TOL = 1e-12
SHAPE = (12, 10, 8)
SCALAR, MATRIX, UPWIND = ("central plus scalar dissipation", "central plus matrix dissipation", "upwind")
DISCS = {"scalar": SCALAR, "matrix": MATRIX, "upwind": UPWIND}
# ADFB_TILE=9,5,4: tiles start at i = 2 + 8 b, j = 2 + 4 b, k chunks at 2 + 4 b (tests/test_regimes_gpu.py); the faces
# 9|10, 5|6 and 5|6 are seams, and the hole / fringe boundary of overset_layout(at=SEAMS) lies on each
TILE, SEAMS = "9,5,4", (9, 5, 5)
SA_TILE = "7,4,3"          # ADFB_SA_TILE: i tiles from 2 + 7 b, j from 2 + 4 b, k chunks of 3 (tests/sa_configs.py)


def _blanked(shape, options=None, at=(5, 5, 5), **kw):
    """(prm, blanked block, the same block without blanking and porosities)"""
    prm, hb = case(*shape, options, **kw)
    plain = hb.copy()
    overset_layout(hb, at)
    return prm, hb, plain


def _moves(a, a0, tol, what):
    moved = rel_l2(a, a0)
    assert moved > 1e3 * tol, "%s: the blanking moves it by %.3e only" % (what, moved)


def _rows(hb, got, want, rows, tol, what):
    ow = hb.d.owned()
    for l in rows:
        a, b = got[ow + (l,)], want[ow + (l,)]
        assert np.isfinite(a).all(), (what, l)
        assert rel_l2(a, b) < tol, "%s[%d] rel L2 %.3e" % (what, l, rel_l2(a, b))
        assert rel_max(a, b) < 10 * tol, "%s[%d] rel max %.3e" % (what, l, rel_max(a, b))


# ---------------------------------------------------------------------------------------------------------------------
# a. full residual
def _oracle_full_residual(prm, hb, flags, preamble):
    if not preamble:
        return oracle_residual(prm, hb, flags)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(flags)
    return ho


def _device_residual(prm, hb, flags, env):
    with _env(**env):
        s = ADFLOW_B200(prm)
        try:
            s.addBlock(hb)
            if flags & RES_DISS_APPROX:
                s.referenceShockSensor()
            s.residual(flags)
            return s.downloadResidual(0), s.downloadIntermed(0)
        finally:
            s.close()


RESIDUAL_CASES = [(d, f, "host", False) for d in DISCS for f in ("exact", "approx")] + [
    (d, "exact", "host", True) for d in DISCS] + [
    ("scalar", "exact", "tile_seams", False), ("scalar", "exact", "tile_seams", True),      # the tile kernel: exact scalar only
    ("scalar", "exact", "sa_seams", False), ("upwind", "exact", "sa_seams", True)]


@pytest.mark.parametrize("disc,fluxes,tiles,preamble", RESIDUAL_CASES, ids=["-".join(map(str, c)) for c in RESIDUAL_CASES])
def test_residual(cuda_lib, disc, fluxes, tiles, preamble):
    env = {"host": {"ADFB_TILE": None, "ADFB_SA_TILE": None}, "tile_seams": {"ADFB_TILE": TILE, "ADFB_SA_TILE": None},
           "sa_seams": {"ADFB_TILE": None, "ADFB_SA_TILE": SA_TILE}}[tiles]
    shape = (16, 12, 11) if tiles == "sa_seams" else SHAPE
    prm, hb, plain = _blanked(shape, {"discretization": DISCS[disc]}, at=SEAMS if tiles == "tile_seams" else (8, 5, 4))
    flags = RES_FLOW | RES_TURB
    if fluxes == "approx":
        flags |= RES_DISS_APPROX | RES_VISC_APPROX
        for h in (hb, plain):
            Oracle(h, prm).reference_shock_sensor()
    ref = _oracle_full_residual(prm, hb, flags, preamble)
    ref0 = _oracle_full_residual(prm, plain, flags, preamble)
    dw, inter = _device_residual(prm, hb, flags | (0 if preamble else RES_SKIP_PREAMBLE), env)
    _rows(hb, dw, ref.dw, range(6), TOL, "dw")
    d, ow = hb.d, hb.d.owned()
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    for n in ("radI", "radJ", "radK"):
        assert rel_max(inter[n], getattr(ref, n)[c1]) < TOL, n
    assert rel_max(inter["dtl"][1:-1, 1:-1, 1:-1], ref.dtl[ow]) < TOL
    for l in range(6):
        _moves(ref.dw[ow + (l,)], ref0.dw[ow + (l,)], TOL, "dw[%d]" % l)
    assert (dw[ow][hb.iblank[ow] <= 0] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# b. smoother residual, stages of rFil = 1.0, 0.56, 0.44
def _oracle_smoother_stages(prm, hb, stages):
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    out = []
    for st in stages:
        o.residual_block(prm.cdisRK[st])
        out.append((ho.dw.copy(), ho.fw.copy()))
    return ho, out


@pytest.mark.parametrize("disc", list(DISCS))
def test_smoother_residual(cuda_lib, disc):
    """k_faces / k_div, or with ADFB_FUSED_SMOOTHER=1 in the process environment the tile kernel for the scalar scheme
    (the library reads the variable once per process: test_smoother_residual_in_the_tile_kernel)"""
    prm, hb, plain = _blanked(SHAPE, {"discretization": DISCS[disc], "nRKStages": 5}, at=(6, 5, 4))
    stages = [st for st in range(5) if prm.cdisRK[st] != 0.0]
    assert [prm.cdisRK[st] for st in stages] == [1.0, 0.56, 0.44]
    ho, ref = _oracle_smoother_stages(prm, hb, stages)
    _, ref0 = _oracle_smoother_stages(prm, plain, stages)
    got = []
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        inter = s.downloadIntermed(0)
        for st in stages:
            s.smootherResidual(st)
            got.append((s.downloadResidual(0), s.downloadArray(0, "fw", 5)))
    finally:
        s.close()
    d, ow = hb.d, hb.d.owned()
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    if disc == "scalar":
        for n in ("radI", "radJ", "radK"):
            assert rel_max(inter[n], getattr(ho, n)[c1]) < TOL, n
    assert rel_max(inter["dtl"][1:-1, 1:-1, 1:-1], ho.dtl[ow]) < TOL
    blank = hb.iblank[ow] <= 0
    for st, (dw, fw), (dwo, fwo), (dw0, fw0) in zip(stages, got, ref, ref0):
        _rows(hb, dw, dwo, range(5), TOL, "dw at stage %d" % st)
        _rows(hb, fw, fwo, range(5), TOL, "fw at stage %d" % st)
        assert (dw[ow][..., :5][blank] == 0).all()
        _moves(dwo[ow][..., :5], dw0[ow][..., :5], TOL, "dw at stage %d" % st)
        _moves(fwo[ow], fw0[ow], TOL, "fw at stage %d" % st)


@pytest.mark.skipif(os.environ.get("ADFB_FUSED_SMOOTHER") == "1", reason="already the ADFB_FUSED_SMOOTHER=1 run")
def test_smoother_residual_in_the_tile_kernel(cuda_lib):
    """the scalar smoother residual with the tile kernel's smoother form (ADFB_FUSED_SMOOTHER=1), which the library
    selects once per process: a process of its own"""
    env = dict(os.environ, ADFB_FUSED_SMOOTHER="1")
    here = os.path.dirname(os.path.abspath(__file__))
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.join(here, "test_blanking_gpu.py") + "::test_smoother_residual[scalar]",
                        "-m", "gpu", "-q", "-p", "no:cacheprovider"], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "1 passed" in r.stdout, r.stdout[-3000:] + r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------------
# c. / d. / e. smoothers: RK cycle, DADI step and cycle, SA DD-ADI
def _smoother_start(prm, hb):
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(prm.cdisRK[0])
    return ho, o


def _device_smoother(prm, hb, run):
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        run(s)
        return s.downloadState(0)
    finally:
        s.close()


def _state_change(hb, w, wo, w0o, tol, rows=range(5)):
    """device state change against the oracle's (rel L2 < tol per row), and the blanking moves the oracle's by 1e3 tol"""
    ow = hb.d.owned()
    for l in rows:
        dv, do = w[ow + (l,)] - hb.w[ow + (l,)], wo[ow + (l,)] - hb.w[ow + (l,)]
        assert np.abs(do).max() > 0
        assert rel_l2(dv, do) < tol, ("state change", l, rel_l2(dv, do))
        _moves(do, w0o[ow + (l,)] - hb.w[ow + (l,)], tol, "state change[%d]" % l)


def _blanked_cells_kept(hb, w, rows):
    ow = hb.d.owned()
    blank = hb.iblank[ow] <= 0
    for l in rows:
        assert np.array_equal(w[ow + (l,)][blank], hb.w[ow + (l,)][blank]), "row %d of a blanked cell changed" % l


@pytest.mark.parametrize("avg", ["never", "always", "alternate"])
def test_rk_cycle(cuda_lib, avg):
    prm, hb, plain = _blanked((16, 12, 10), {"nRKStages": 5, "resAveraging": avg}, at=(7, 5, 4))
    ho, o = _smoother_start(prm, hb)
    o.rk_smoother()
    h0, o0 = _smoother_start(prm, plain)
    o0.rk_smoother()
    w, p, rlv, rev = _device_smoother(prm, hb, lambda s: s.rkCycle())
    _state_change(hb, w, ho.w, h0.w, 1e-10)
    assert rel_max(p, ho.p) < 1e-11
    if avg == "never":       # residual averaging couples an unblanked neighbour's epz into a blanked row
        _blanked_cells_kept(hb, w, [0])
        _blanked_cells_kept(hb, ho.w, [0])


@pytest.mark.parametrize("shape,at", [((14, 11, 9), (6, 5, 4)), ((118, 119, 3), (30, 32, 2))],
                         ids=["14x11x9", "long-lines-118x119x3"])
@pytest.mark.parametrize("entry", ["step", "cycle"])
def test_dadi(cuda_lib, shape, at, entry):
    """(118, 119, 3): 119 x 3 i lines, in groups of 32 in the tiled i sweep; the fringe shell at j = 31 .. 36 spans the
    line groups 0 | 1 of the k = 2 plane"""
    prm, hb, plain = _blanked(shape, {"smoother": "DADI"}, at=at)

    def oracle(h):
        ho, o = _smoother_start(prm, h)
        o.dadi_step()
        if entry == "cycle":
            o.residual_block(1.0)
            o.dadi_step()
        return ho

    ho, h0 = oracle(hb), oracle(plain)
    w, p, rlv, rev = _device_smoother(prm, hb, (lambda s: s.dadiStep()) if entry == "step" else (lambda s: s.dadiCycle(2)))
    _state_change(hb, w, ho.w, h0.w, 1e-9)
    assert rel_max(p, ho.p) < 1e-11
    _blanked_cells_kept(hb, w, [0])
    _blanked_cells_kept(hb, ho.w, [0])


@pytest.mark.parametrize("niter", [1, 3])
@pytest.mark.parametrize("shape,at", [(SHAPE, (6, 5, 4)), ((40, 18, 17), (11, 9, 8))], ids=["12x10x8", "40x18x17"])
def test_sa_ddadi(cuda_lib, shape, at, niter):
    """(40, 18, 17): lines of 16 cells or more run the 8-lane partitioned line solve; the shell crosses its partitions"""
    prm, hb, plain = _blanked(shape, at=at)

    def oracle(h):
        ho = h.copy()
        o = Oracle(ho, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        for _ in range(niter):
            o.sa_block()
        return ho

    ho, h0 = oracle(hb), oracle(plain)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.turbSolveDDADI(niter)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    _state_change(hb, w, ho.w, h0.w, 1e-9, rows=[5])
    assert rel_max(w[..., 5], ho.w[..., 5]) < 1e-10
    d = hb.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    assert rel_max(rev[c1], ho.rev[c1]) < 1e-10
    _blanked_cells_kept(hb, w, [5])
    _blanked_cells_kept(hb, ho.w, [5])


# ---------------------------------------------------------------------------------------------------------------------
# f. matrix-free and ANK products
def _state_vec(hb):
    return np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()


def _slab_seam_layout(hb):
    """the form-function pipeline cuts k into slabs at chunks of 4 planes (cells 2 + 4 c): noFlux on part of every face
    k = 1 + 4 c and a hole / fringe pair across it"""
    d = hb.d
    for k in range(5, d.kl, 4):
        hb.porK[2:d.il // 2, 2:d.jl // 2, k] = -1
        hb.iblank[d.il - 3:d.il - 1, 2:4, k] = 0
        hb.iblank[d.il - 3:d.il - 1, 2:4, k + 1] = -1


def test_form_function_and_mffd(cuda_lib):
    import torch

    prm, hb, plain = _blanked((16, 12, 48), at=(6, 5, 8))
    _slab_seam_layout(hb)
    U = _state_vec(hb) * (1.0 + 1e-3 * np.random.default_rng(3).standard_normal(hb.d.ncells * hb.nw))
    a = np.random.default_rng(5).standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-7
    ref, ref1 = oracle_form_function(prm, hb, U), oracle_form_function(prm, hb, U + h * a)
    _moves(ref, oracle_form_function(prm, plain, U), TOL, "form function")
    s = ADFLOW_B200(prm)
    pipes = {}
    try:
        s.addBlock(hb)
        r = s.formFunction(U)
        n = s.getStateSize()
        hw, hr = (torch.empty(n, dtype=torch.float64).pin_memory() for _ in range(2))
        hw.numpy()[:] = U
        for slabs in ("3", "6"):
            hr.numpy()[:] = np.nan
            with _env(ADFB_FF_PIPE=slabs):
                s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
            pipes[slabs] = hr.numpy().copy()
        s.mffdSetBase(U)
        y = s.mffdApply(a, h)
        ad = torch.from_numpy(a).cuda()
        yd = torch.empty_like(ad)
        s.mffdApplyDevice(ad.data_ptr(), yd.data_ptr(), n, h)
        y_dev = yd.cpu().numpy()
    finally:
        s.close()
    assert rel_l2(r, ref) < TOL, rel_l2(r, ref)
    for slabs, rp in pipes.items():
        assert np.isfinite(rp).all() and rel_l2(rp, ref) < 1e-11, (slabs, rel_l2(rp, ref))
    yref = (ref1 - ref) / h
    assert rel_l2(y, yref) < 1e-4, rel_l2(y, yref)
    assert rel_l2(y_dev, yref) < 1e-4, rel_l2(y_dev, yref)


@pytest.mark.parametrize("coupled", [False, True])
def test_ank_operator_and_product(cuda_lib, coupled):
    """adfb_ank_form_function and the ANK product (approximate fluxes, as tests/test_ank_gpu.py); the physicality check
    works on the vectors alone and reads no blanking"""
    prm, hb, plain = _blanked((14, 11, 9), at=(6, 5, 4))
    ank = make_ank_params(cfl=5.0, coupled=coupled, char_time_step="VLR", mach=0.8, cflLimit=50.0, turbCFLScale=2.0)
    ns = hb.nw if coupled else 5
    h = 1e-6
    ops = {}
    for name, blk in (("blanked", hb), ("plain", plain)):
        o = Oracle(blk, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        o.time_step(True)
        o.call("orc_speed_of_sound", C.byref(prm))
        o.reference_shock_sensor()
        T = oracle_blocks(prm, ank, blk)
        U = vec_of(blk, ns)
        rng = np.random.default_rng(5)
        v = U * (1.0 + 0.01 * rng.standard_normal(U.size))
        a = rng.standard_normal(U.size) * np.abs(U).clip(1e-6)
        F0 = oracle_ank_function(prm, ank, blk, T, U)
        ops[name] = (U, v, a, oracle_ank_function(prm, ank, blk, T, v), (oracle_ank_function(prm, ank, blk, T, U + h * a) - F0) / h)
    U, v, a, Fref, yref = ops["blanked"]
    # the product's finite-difference tolerance is too loose for the blanking to move it 1e3 times; the function it
    # differences carries the sensitivity check
    _moves(Fref, ops["plain"][3], TOL, "ANK function")
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        s.referenceShockSensor()
        s.residual(RES_FLOW | RES_TURB | 4)        # useUpdateIntermed: dtl, spectral radii of the current state
        s.ankTimeStepMat()
        F = s.ankFormFunction(v)
        s.ankMffdSetBase(U)
        y = s.ankMffdApply(a, h)
    finally:
        s.close()
    assert rel_l2(F, Fref) < 1e-11, rel_l2(F, Fref)
    assert rel_l2(y, yref) < 1e-5, rel_l2(y, yref)


def _oracle_turb_function(prm, ank, hb, v):
    """FormFunction_mf_turb of the decoupled ANK with the oracle, as tests/test_ank_gpu.py composes it"""
    ow = hb.d.owned()
    h2 = hb.copy()
    o = Oracle(h2, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    dtl = h2.dtl.copy()
    h2.w[ow + (5,)] = np.transpose(v.reshape(hb.d.nz, hb.d.ny, hb.d.nx), (2, 1, 0))
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, hb.d.il, 2, hb.d.jl, 2, hb.d.kl)
    o.residual_core(RES_TURB)
    h2.dtl[...] = dtl
    r = np.empty_like(v)
    o.L.orc_ank_turb_rvec(C.byref(o.ob), C.byref(prm), C.byref(ank), v.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p))
    return r


def test_turbulence_ksp_pieces(cuda_lib):
    """adfb_ank_form_function_turb and its product: the SA row of the residual is multiplied by max(iblank, 0)"""
    prm, hb, plain = _blanked((12, 9, 8), at=(6, 4, 3))
    ank = make_ank_params(cfl=5.0, coupled=False, physLSTolTurb=0.99, stepMin=0.01, stepFactor=1.0)
    ow = hb.d.owned()
    U = np.ascontiguousarray(np.transpose(hb.w[ow][..., 5], (2, 1, 0)).reshape(-1))
    rng = np.random.default_rng(5)
    vin = U * (1.0 + 0.01 * rng.standard_normal(U.size))
    a = rng.standard_normal(U.size) * np.abs(U)
    h = 1e-6
    want = _oracle_turb_function(prm, ank, hb, vin)
    _moves(want, _oracle_turb_function(prm, ank, plain, vin), 1e-11, "turbulence function")
    yref = (_oracle_turb_function(prm, ank, hb, U + h * a) - _oracle_turb_function(prm, ank, hb, U)) / h
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        s.residual(RES_FLOW | RES_TURB | 4)
        r = s.ankFormFunctionTurb(vin)
        s.ankMffdTurbSetBase(U)
        y = s.ankMffdTurbApply(a, h)
    finally:
        s.close()
    assert rel_l2(r, want) < 1e-11, rel_l2(r, want)
    assert rel_l2(y, yref) < 1e-6, rel_l2(y, yref)


def _blanked_rows(hb):
    """mask of the entries of a state vector (cell-major, nw per cell) that belong to cells with iblank <= 0"""
    return np.repeat(np.transpose(hb.iblank[hb.d.owned()] <= 0, (2, 1, 0)).reshape(-1), hb.nw)


def _gmres_nk(prm, hb):
    from test_ank_gpu import _host_gmres

    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        U = s.getStates()
        s.mffdSetBase(U)
        apply = lambda v: s.mffdApply(v, -1.0)  # noqa: E731
        b = apply(np.random.default_rng(3).standard_normal(U.size) * np.abs(U).clip(1e-6) * 1e-3)
        x, its, rn = s.gmresSolve(b, op="NK", restart=10, max_its=10, rtol=1e-3)
        xh, its_h = _host_gmres(apply, b, 10, 10, 1e-3)
    finally:
        s.close()
    return b, x, its, rn, xh, its_h


def test_gmres_nk_on_a_blanked_block(cuda_lib):
    """adfb_gmres_solve op 0 against a host GMRES applying the same device product (tests/test_ank_gpu.py).  The rows of
    cells with iblank <= 0 of every product are exactly zero, so the right-hand side and every Krylov vector are zero
    there, and so is the solution, bit for bit; on the block without blanking those rows carry a sizeable part of it"""
    prm, hb, plain = _blanked((10, 8, 7), at=(4, 4, 3))
    b, x, its, rn, xh, its_h = _gmres_nk(prm, hb)
    assert np.isfinite(x).all() and its >= 1 and abs(its - its_h) <= 1
    assert rn <= np.linalg.norm(b) * (1 + 1e-12)
    assert np.linalg.norm(x - xh) < 2e-2 * np.linalg.norm(xh), np.linalg.norm(x - xh) / np.linalg.norm(xh)
    rows = _blanked_rows(hb)
    assert rows.any() and (b[rows] == 0).all() and (x[rows] == 0).all()
    _, x0, *_ = _gmres_nk(prm, plain)
    assert np.linalg.norm(x0[rows]) > 1e-2 * np.linalg.norm(x0)


# ---------------------------------------------------------------------------------------------------------------------
# g. multigrid: blanked fine level, noFlux / boundFlux planes on every coarse level
def _mg_levels(shape, options, nlev, blanked):
    """the levels of tests/test_mg_gpu.py; blanked: overset_layout on the fine level and, on each coarse level, the
    setPorosities faces of make_coarse_block plus coarse_interior_planes (coarse levels carry no blanking: the
    reference's transfers never read iblank)"""
    from util import coarse_interior_planes

    prm, fine = case(*shape, options)
    if blanked:
        overset_layout(fine, at=(6, 5, 3))
    o = Oracle(fine, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    levels = [fine]
    for _ in range(nlev - 1):
        levels.append(syn.make_coarse_block(levels[-1], prm))
        if blanked:
            coarse_interior_planes(levels[-1])
    return prm, levels


@pytest.mark.parametrize("cycle,options,dadi_sub,tol,wtol", [("2v", None, 0, 1e-8, 1e-10),
                                                             ("3w", {"smoother": "DADI", "resAveraging": "never"}, 2, 1e-7, 1e-9)],
                         ids=["2v-rk", "3w-dadi"])
def test_mg_cycle(cuda_lib, cycle, options, dadi_sub, tol, wtol):
    """tolerances of tests/test_mg_gpu.py"""
    from test_mg_gpu import device, oracle_mg_cycle, prepare_fine

    nlev = int(cycle[0])
    cyc = ADFLOW_B200.cycleStrategy(cycle)
    oracle_w, start = {}, {}
    for blanked in (True, False):
        prm, levels = _mg_levels((16, 12, 8), options, nlev, blanked)
        if blanked:
            dev_levels = [l_.copy() for l_ in levels]
        prepare_fine(Oracle(levels[0], prm))
        start[blanked] = levels[0].w.copy()
        oracle_mg_cycle(prm, levels, cyc, dadi_subiter=dadi_sub)
        oracle_w[blanked] = levels[0]
    fine, w0 = oracle_w[True], start[True]
    s = device(prm, dev_levels)
    try:
        s.timeStep(False)
        s.smootherResidual(0)
        if dadi_sub:
            s.mgCycle(cyc, smoother="DADI", n_subiterations=dadi_sub)
        else:
            s.mgCycle(cyc)
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = fine.d.owned()
    for l in range(5):
        a, b = w[ow + (l,)] - w0[ow + (l,)], fine.w[ow + (l,)] - w0[ow + (l,)]
        assert np.abs(b).max() > 0
        assert rel_l2(a, b) < tol, ("state change over the cycle", l, rel_l2(a, b))
        _moves(b, oracle_w[False].w[ow + (l,)] - start[False][ow + (l,)], tol, "state change over the cycle [%d]" % l)
        if not dadi_sub:
            assert rel_l2(dw[ow + (l,)], fine.dw[ow + (l,)]) < tol, ("residual after the cycle", l)
    assert rel_max(w[..., :5], fine.w[..., :5]) < wtol


# ---------------------------------------------------------------------------------------------------------------------
# h. wall forces weighted by the surface iblank
FORCE_TOL = 1e-11


def _oracle_forces(prm, hb, ref_point, p_ref):
    """forces of the oracle after the residual that stores the wall stresses; the halos made consistent first"""
    o = Oracle(hb, prm)
    if prm.equations == 3:
        o.apply_turb_bc(True)
    o.apply_flow_bc(True)
    ho = hb.copy()
    Oracle(ho, prm).residual_core(RES_FLOW | (RES_TURB if prm.equations == 3 else 0))
    return ho, Oracle(ho, prm).wall_forces(ref_point, p_ref)


def _device_forces(prm, blocks, ref_point, p_ref):
    s = ADFLOW_B200(prm)
    try:
        for hb in blocks:
            s.addBlock(hb)
        s.residual(RES_FLOW | (RES_TURB if prm.equations == 3 else 0) | RES_STORE_WALL | RES_SKIP_PREAMBLE)
        return s.getForces(ref_point, p_ref)
    finally:
        s.close()


def _forces_match(got, want, moved_from):
    scale = np.abs(want).max(axis=1, keepdims=True)
    rows = scale[:, 0] > 0
    assert rows[0] and rows[2]
    assert (np.abs(got - want)[rows] <= FORCE_TOL * scale[rows]).all(), (got - want) / np.where(scale > 0, scale, 1)
    moved = np.abs(want - moved_from).max(axis=1)
    assert (moved[rows] > 1e3 * FORCE_TOL * scale[rows, 0]).all(), moved


@pytest.mark.parametrize("walls", ["adiabatic", "isothermal", "euler", "MIXED"])
def test_wall_forces_surface_iblank(cuda_lib, walls):
    from test_oracle_vs_reference_blanking import WALLS
    from util import volume_weighted

    opts, perm = WALLS[walls]
    if perm is None:
        prm, hb = case(12, 9, 10, opts, split=MIXED)
    else:
        prm, hb = case(12, 9, 10, opts, physical_faces=perm)
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    blank_wall_surfaces(hb)
    ref_point, p_ref = (0.3, -0.2, 0.1), 2.5
    ho, want = _oracle_forces(prm, hb, ref_point, p_ref)
    hv = ho.copy()
    hv.subfaces = volume_weighted(ho)
    by_volume = Oracle(hv, prm).wall_forces(ref_point, p_ref)
    got = _device_forces(prm, [hb], ref_point, p_ref)
    _forces_match(got, want, by_volume)
    if rb.available():
        ref = rb.wall_forces(ho, prm, ref_point, p_ref)
        scale = np.abs(want).max(axis=1, keepdims=True)
        assert (np.abs(got - ref) <= FORCE_TOL * scale).all()


def test_wall_forces_of_several_blocks(cuda_lib):
    """four blocks of different shapes in one context: A with its walls blanked, B with a NULL surface iblank over
    first-layer cells of volume iblank 0 (without overset the wall counts in full, BCData.F90:2182), C with a wall split
    into pieces of different surface blanking (the KMIN pieces carry slices of one face's pattern, the IMIN piece none),
    and D, the last block, whose blanked wall decides the sums"""
    prm = make_params({"equationType": "RANS"})
    ISO = {1: 3, 2: 6, 3: 2, 4: 3, 5: 1, 6: 3}
    A = syn.make_block(24, 16, 12, prm, seed=1101)
    B = syn.make_block(17, 13, 10, prm, seed=2203, physical_faces=ISO)
    C_ = syn.make_block(12, 9, 18, prm, seed=3307)
    D = syn.make_block(9, 7, 11, prm, seed=4409, physical_faces={1: 3, 2: 3, 3: 3, 4: 3, 5: 3, 6: 2})
    blank_wall_surfaces(A)
    for s in B.subfaces:
        if s["bcType"] in (2, 6):
            B.iblank[wall_layer(B, s)] = 0
            assert "iblank" not in s
    blank_wall_surfaces(C_)                       # the KMIN wall, before the split slices it
    split_faces(C_, prm, MIXED)
    assert sum(1 for s in C_.subfaces if s["bcType"] in (2, 6) and "iblank" in s) == 2
    assert any(s["bcType"] in (2, 6) and "iblank" not in s for s in C_.subfaces)
    D.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    blank_wall_surfaces(D)
    D.subfaces[0]["iblank"][...] = 0              # D's wall blanked but for one face cell, which decides the sums
    D.subfaces[0]["iblank"][5, 6] = 1
    blocks = [A, B, C_, D]
    for hb in blocks:
        hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (2, 6) else 1)
    ref_point, p_ref = (0.3, -0.2, 0.1), 2.5
    want, full = np.zeros((4, 3)), np.zeros((4, 3))
    for hb in blocks:
        ho, f = _oracle_forces(prm, hb, ref_point, p_ref)
        want += f
        hv = ho.copy()
        for s in hv.subfaces:
            s.pop("iblank", None)
        full += Oracle(hv, prm).wall_forces(ref_point, p_ref)
    got = _device_forces(prm, blocks, ref_point, p_ref)
    _forces_match(got, want, full)
    # without D the sums differ by more than the tolerance: the last block is read
    got3 = _device_forces(prm, blocks[:3], ref_point, p_ref)
    scale = np.abs(want).max(axis=1, keepdims=True)
    assert (np.abs(got3 - got).max(axis=1)[:2] > 1e3 * FORCE_TOL * scale[:2, 0]).all()
