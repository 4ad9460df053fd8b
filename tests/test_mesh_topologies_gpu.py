"""The device path on the meshes of tests/meshes.py, against the oracle: an O-grid whose j faces are one periodic cut
of the block with itself (a same-block 1-to-1 exchange), a polar grid whose kMin face is collapsed onto the axis (zero
face areas, wedge cells, the polar BC on a singular line), and the O-grid with its stiff wall-normal direction along j
and along i instead of k, where the tile kernel's i-j tiles, the tiled DADI i sweep and the partitioned SA line solves
meet aspect ratios of 1e4 and more.

Tolerances are those of the existing tests of each entry point (test_residual_parity.py, test_smoother_parity.py,
test_dadi.py, test_sa_solve.py, test_forces.py, test_form_function_pipeline.py).  The device equivariance test holds the
device to ten times the oracle's own measured equivariance (test_mesh_topologies_host.py)."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from adflow_b200 import make_params
from adflow_b200.halo import exchange_numpy
from adflow_b200.solver import ADFLOW_B200, RES_DISS_APPROX, RES_FLOW, RES_SKIP_PREAMBLE, RES_STORE_WALL, RES_TURB, RES_VISC_APPROX
from oracle.pyoracle import Oracle

import meshes
from test_mesh_topologies_host import ORACLE_EQUIVARIANCE_DTL, ORACLE_EQUIVARIANCE_DW
from test_residual_parity import compare
from test_sa_tile_gpu import _env
from util import rel_l2, rel_max

pytestmark = pytest.mark.gpu

GENERAL_KERNELS = os.environ.get("ADFB_FUSED") == "0"
SCALAR, MATRIX, UPWIND = ("central plus scalar dissipation", "central plus matrix dissipation", "upwind")
DISCS = {"scalar": SCALAR, "matrix": MATRIX, "upwind": UPWIND}
PERM = {"o_grid": (0, 1, 2), "o_grid_jk": (1, 2, 0), "o_grid_ki": (2, 0, 1)}
BLOCKS = [("o_grid", "Euler"), ("o_grid", "laminar NS"), ("o_grid", "RANS"), ("polar", "RANS"), ("o_grid_jk", "RANS"),
          ("o_grid_ki", "RANS")]
IDS = ["%s-%s" % (n, e.split()[0]) for n, e in BLOCKS]


def block(name, eq="RANS", options=None, shape=(10, 12, 8), **mesh_kw):
    """(prm, block, its periodic pattern of the finest level); shape: the unpermuted block's (axial, circumferential,
    radial) cell counts"""
    opts = {"equationType": eq}
    opts.update(options or {})
    prm = make_params(opts)
    if name == "polar":
        hb, axis = meshes.polar_grid(*shape, prm, **mesh_kw), 1
    else:
        perm = PERM[name]
        hb, axis = meshes.permute_axes(meshes.o_grid(*shape, prm, **mesh_kw), perm), meshes.inverse(perm)[1]
    return prm, hb, meshes.self_periodic_pattern(hb, 2, axis)


def flags_of(prm):
    return RES_FLOW | (RES_TURB if prm.equations == 3 else 0)


def box_close(a, b, tol, name):
    assert np.isfinite(a).all(), name
    err = rel_max(a, b)
    assert err < tol, "%s: rel max %.3e" % (name, err)


def compare_core(prm, hb, flags):
    """test_residual_parity.compare (dw rows, radii and dtl against the oracle), and every array it downloads finite,
    halos included"""
    ref, dw, norms, extra = compare(prm, hb, flags)
    for n, a in [("dw", dw)] + list(extra.items()):
        assert np.isfinite(a).all(), n
    assert np.isfinite(norms).all()


# ---------------------------------------------------------------------------------------------------------------------
# residual core (RES_SKIP_PREAMBLE): the state handed out is already consistent across the cut
@pytest.mark.parametrize("name,eq", BLOCKS, ids=IDS)
@pytest.mark.parametrize("disc", list(DISCS))
@pytest.mark.parametrize("fluxes", ["exact", "approx"])
def test_residual_core(cuda_lib, name, eq, disc, fluxes):
    prm, hb, _ = block(name, eq, {"discretization": DISCS[disc]})
    flags = flags_of(prm)
    if fluxes == "approx":
        flags |= RES_DISS_APPROX | RES_VISC_APPROX
        Oracle(hb, prm).reference_shock_sensor()
    compare_core(prm, hb, flags)


# ADFB_TILE=9,5,4: tile seams at i = 9|10, j = 5|6, k chunks from 2 + 4 b; ADFB_SA_TILE=7,4,3: SA tiles from 2 + 7 b in i,
# 2 + 4 b in j, k chunks of 3.  On o_grid_ki the wall-normal direction is i, on o_grid_jk j, on o_grid k: every seam
# cuts the stiff direction on one of them.
@pytest.mark.skipif(GENERAL_KERNELS, reason="tile kernels only")
@pytest.mark.parametrize("name", ["o_grid", "o_grid_jk", "o_grid_ki", "polar"])
@pytest.mark.parametrize("env", [{"ADFB_TILE": "9,5,4", "ADFB_SA_TILE": None}, {"ADFB_TILE": None, "ADFB_SA_TILE": "7,4,3"}],
                         ids=["tile_seams", "sa_seams"])
def test_residual_core_tile_seams(cuda_lib, name, env):
    prm, hb, _ = block(name, shape=(17, 12, 11))
    with _env(**env):
        compare_core(prm, hb, RES_FLOW | RES_TURB)


@pytest.mark.skipif(GENERAL_KERNELS, reason="already the ADFB_FUSED=0 run")
def test_general_kernels_still_match(cuda_lib):
    """the same file with the general kernels (ADFB_FUSED=0) in place of the tile kernel"""
    env = dict(os.environ, ADFB_FUSED="0")
    r = subprocess.run([sys.executable, "-m", "pytest", os.path.abspath(__file__), "-m", "gpu", "-q", "-x"], env=env,
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


# ---------------------------------------------------------------------------------------------------------------------
# full residual: state preparation, BCs (the polar one on the collapsed face), the periodic self-exchange, owned rhoE
def oracle_full_residual(prm, hb, pat, flags):
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    exchange_numpy([ho], pat, meshes.state_vars)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(flags)
    return ho


@pytest.mark.parametrize("name,eq", BLOCKS, ids=IDS)
def test_full_residual_with_preamble(cuda_lib, name, eq):
    prm, hb, pat = block(name, eq)
    own = hb.d.owned() + (slice(0, 5),)
    hb.w[own] *= 1.0 + 1e-3 * np.random.default_rng(5).standard_normal(hb.w[own].shape)   # the cut's halos are stale now
    flags = flags_of(prm)
    ho = oracle_full_residual(prm, hb, pat, flags)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.setCommPattern(pat)
        s.residual(flags)
        dw = s.downloadResidual(0)
        w, p, rlv, rev = s.downloadState(0)
        inter = s.downloadIntermed(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(hb.nw if flags & RES_TURB else 5):
        assert np.isfinite(dw[ow + (l,)]).all()
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-12, (l, rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]))
    for a, b, n in ((w, ho.w, "w"), (p, ho.p, "p"), (rlv, ho.rlv, "rlv"), (rev, ho.rev, "rev")):
        box_close(a, b, 1e-13, n)     # every halo: BCs, the cut, the edges of both
    for n, a in inter.items():
        assert np.isfinite(a).all(), n


# ---------------------------------------------------------------------------------------------------------------------
# smoothers.  One block without a communication pattern on both sides: the stages are compared on this geometry (the
# state is consistent across the cut when they start); the exchange inside a cycle is tested by the full residual above.
@pytest.mark.parametrize("name,eq", BLOCKS, ids=IDS)
@pytest.mark.parametrize("disc", list(DISCS))
def test_smoother_residual(cuda_lib, name, eq, disc):
    prm, hb, _ = block(name, eq, {"discretization": DISCS[disc], "nRKStages": 5})
    stages = [st for st in range(5) if prm.cdisRK[st] != 0.0]
    assert [prm.cdisRK[st] for st in stages] == [1.0, 0.56, 0.44]
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        inter = s.downloadIntermed(0)
        d, ow = hb.d, hb.d.owned()
        assert rel_max(inter["dtl"][1:-1, 1:-1, 1:-1], ho.dtl[ow]) < 1e-12
        c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
        if disc == "scalar":
            for n in ("radI", "radJ", "radK"):
                assert rel_max(inter[n], getattr(ho, n)[c1]) < 1e-12, n
        for st in stages:
            o.residual_block(prm.cdisRK[st])
            s.smootherResidual(st)
            dw, fw = s.downloadResidual(0), s.downloadArray(0, "fw", 5)
            for l in range(5):
                for a, b, what in ((dw, ho.dw, "dw"), (fw, ho.fw, "fw")):
                    assert np.isfinite(a[ow + (l,)]).all()
                    assert rel_l2(a[ow + (l,)], b[ow + (l,)]) < 1e-12, (st, what, l, rel_l2(a[ow + (l,)], b[ow + (l,)]))
    finally:
        s.close()


@pytest.mark.parametrize("name", ["o_grid", "polar", "o_grid_jk", "o_grid_ki"])
@pytest.mark.parametrize("avg", ["never", "always", "alternate"])
def test_rk_cycle(cuda_lib, name, avg):
    prm, hb, _ = block(name, options={"nRKStages": 5, "resAveraging": avg})
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(prm.cdisRK[0])
    o.rk_smoother()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        s.rkCycle()
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    ow = hb.d.owned()
    dwv, dwo = w[ow] - hb.w[ow], ho.w[ow] - hb.w[ow]
    assert np.abs(dwo[..., :5]).max() > 1e-8
    for l in range(5):
        assert rel_l2(dwv[..., l], dwo[..., l]) < 1e-10, ("state change", l, rel_l2(dwv[..., l], dwo[..., l]))
    box_close(w[..., :5], ho.w[..., :5], 1e-11, "w after the RK cycle (halos included)")
    box_close(p, ho.p, 1e-11, "p after the RK cycle")


# 19 radial cells: the stiff lines of each orientation are three 8-cell chunks of the DADI line walk, the last one short
DADI_CASES = [c + ((10, 12, 8),) for c in BLOCKS] + [(n, "RANS", (10, 12, 19)) for n in PERM]
DADI_IDS = IDS + ["%s-RANS-19" % n for n in PERM]


@pytest.mark.parametrize("name,eq,shape", DADI_CASES, ids=DADI_IDS)
def test_dadi_step(cuda_lib, name, eq, shape):
    prm, hb, _ = block(name, eq, shape=shape)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(1.0)
    o.dadi_step()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        s.dadiStep()
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-10, ("dw after DADI", l)
    dwv, dwo = w[ow] - hb.w[ow], ho.w[ow] - hb.w[ow]
    for l in range(5):
        assert rel_l2(dwv[..., l], dwo[..., l]) < 1e-9, ("state change", l)
    box_close(p, ho.p, 1e-11, "p")
    assert np.isfinite(w).all()


# The SA line solves take the partitioned Thomas solver (k_sa_thomas_part) on lines of 16 .. 256 owned cells
# (adfb_part_lanes): 8 lanes of up to 12 cells each up to 96 cells, 8 lanes of 16 up to 128, 16 lanes of 16 above.  So
# the radial (stiff) lines of each orientation get 20, 110 and 140 cells; the other lines stay shorter than 16.
SA_PART = {20: "k_sa_thomas_part<8,12>", 110: "k_sa_thomas_part<8,16>", 140: "k_sa_thomas_part<16,16>"}
SA_CASES = [("o_grid", 8), ("polar", 8), ("o_grid_jk", 8), ("o_grid_ki", 8)] + [(n, nr) for n in PERM for nr in SA_PART]


@pytest.mark.parametrize("name,radial", SA_CASES, ids=["%s-%d" % c for c in SA_CASES])
def test_sa_ddadi(cuda_lib, name, radial):
    prm, hb, _ = block(name, shape=(10, 12, 8) if radial == 8 else (6, 8, radial))
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    for _ in range(2):
        o.sa_block()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.turbSolveDDADI(2)
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    assert rel_l2(dw[ow + (5,)], ho.dw[ow + (5,)]) < 1e-10
    dn, do = w[ow + (5,)] - hb.w[ow + (5,)], ho.w[ow + (5,)] - hb.w[ow + (5,)]
    assert np.abs(do).max() > 0
    assert rel_l2(dn, do) < 1e-9, rel_l2(dn, do)
    box_close(w[..., 5], ho.w[..., 5], 1e-10, "nuTilde (halos included)")
    d = hb.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    box_close(rev[c1], ho.rev[c1], 1e-10, "rev")


def test_stiff_lines_take_the_partitioned_and_chunked_solves(cuda_lib, tmp_path):
    """test_sa_ddadi and test_dadi_step on the long radial lines, traced one launch at a time (tests/kernel_trace.py, as
    test_dispatch_gpu.py runs it): each SA case launches the partitioned Thomas variant its radial line length selects,
    and the DADI step with 19 radial cells along i launches the tiled, chunked i walk"""
    import json

    here = os.path.dirname(os.path.abspath(__file__))
    sa = {"%s::test_sa_ddadi[%s-%d]" % (os.path.abspath(__file__), n, nr): SA_PART[nr] for n, nr in SA_CASES if nr in SA_PART}
    dadi = "%s::test_dadi_step[o_grid_ki-RANS-19]" % os.path.abspath(__file__)
    out = tmp_path / "trace.json"
    env = dict(os.environ, ADFB_NO_GRAPH="1")
    env["PYTHONPATH"] = os.pathsep.join([here] + ([env["PYTHONPATH"]] if env.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-m", "pytest", "-p", "kernel_trace", "--kernel-trace", str(out), "-q",
                        "-p", "no:cacheprovider", "--rootdir", os.path.dirname(here)] + sorted(sa) + [dadi],
                       cwd=os.path.dirname(here), env=env, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    with open(out) as f:
        seen = json.load(f)

    def traced(node):
        hits = [v for k, v in seen.items() if node.endswith(k) or k.endswith(node.split("::", 1)[1])]
        assert hits, "%s did not run" % node
        return set().union(*map(set, hits))

    for node, kernel in sa.items():
        assert kernel in traced(node), (node, kernel, sorted(traced(node)))
    assert "k_dadi_thomas_tile" in traced(dadi), sorted(traced(dadi))


# ---------------------------------------------------------------------------------------------------------------------
# form function: the slab pipeline does not take blocks with exchange partners, so a call that asks for it takes the
# one-shot path and gives the same bits
def oracle_form_function_cut(prm, hb, pat, U):
    """the oracle's FormFunction_mf with the exchange: setW, preamble, BCs, whalo2, owned rhoE, core, setRVec"""
    d, ow = hb.d, hb.d.owned()
    h2 = hb.copy()
    v = U.reshape(d.nz, d.ny, d.nx, hb.nw).transpose(2, 1, 0, 3).copy()
    v[..., 5] = np.maximum(1e-6 * prm.wInf[5], v[..., 5])
    h2.w[ow] = v
    ho = oracle_full_residual(prm, h2, pat, RES_FLOW | RES_TURB)
    r = ho.dw[ow] / ho.volRef[ow][..., None]
    r[..., 5] *= prm.turbResScale
    return np.transpose(r, (2, 1, 0, 3)).reshape(-1)


def state_vec(hb, seed):
    U = np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()
    return U * (1.0 + 1e-3 * np.random.default_rng(seed).standard_normal(U.size))


def test_form_function_with_the_cut_takes_the_one_shot_path(cuda_lib):
    import torch

    prm, hb, pat = block("o_grid", shape=(8, 12, 16))
    d = hb.d
    U = state_vec(hb, 3)
    want = oracle_form_function_cut(prm, hb, pat, U)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.setCommPattern(pat)
        n = s.getStateSize()
        hw, hr = (torch.empty(n, dtype=torch.float64).pin_memory() for _ in range(2))
        hw.numpy()[:] = U
        with _env(ADFB_FF_PIPE="0"):
            s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        one = hr.numpy().copy()
        hr.numpy()[:] = np.nan
        with _env(ADFB_FF_PIPE="4"):
            s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        asked = hr.numpy().copy()
    finally:
        s.close()
    assert np.isfinite(one).all()
    assert np.array_equal(asked, one)
    got, exp = (np.transpose(x.reshape(d.nz, d.ny, d.nx, hb.nw), (2, 1, 0, 3)) for x in (one, want))
    for l in range(hb.nw):
        assert rel_l2(got[..., l], exp[..., l]) < 1e-11, (l, rel_l2(got[..., l], exp[..., l]))


@pytest.mark.parametrize("name", ["o_grid", "polar", "o_grid_ki"])
def test_mffd_product_with_the_cut(cuda_lib, name):
    """the NK matrix-free product with the cut's exchange inside each residual: against the oracle's difference quotient
    at the tolerance of test_mffd.py, and, with ADFB_MFFD_FUSED=1, the fused form (the perturbation formed inside the
    residual launch) bit for bit the three-pass form, as documented for it"""
    prm, hb, pat = block(name)
    U = state_vec(hb, 3)
    a = np.random.default_rng(314).standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-6
    yref = (oracle_form_function_cut(prm, hb, pat, U + h * a) - oracle_form_function_cut(prm, hb, pat, U)) / h
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.setCommPattern(pat)
        s.mffdSetBase(U)
        y = s.mffdApply(a, h).copy()
        with _env(ADFB_MFFD_FUSED="1"):
            yf = s.mffdApply(a, h).copy()
        y2 = s.mffdApply(a, h).copy()
    finally:
        s.close()
    assert np.isfinite(y).all()
    assert np.array_equal(y, y2)
    assert np.array_equal(yf, y)
    assert rel_l2(y, yref) < 1e-6, rel_l2(y, yref)


# ---------------------------------------------------------------------------------------------------------------------
# wall forces on the cylinder (curved normals) and on the disc of the polar grid
def _device_forces(prm, hb, ref_point, p_ref):
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.residual(RES_FLOW | RES_TURB | RES_STORE_WALL | RES_SKIP_PREAMBLE)
        return s.getForces(ref_point, p_ref)
    finally:
        s.close()


def test_wall_forces(cuda_lib):
    ref_point, p_ref = (0.3, -0.2, 0.1), 2.5
    got = {}
    for name in ("o_grid", "o_grid_jk", "o_grid_ki", "polar"):
        prm, hb, _ = block(name)
        o = Oracle(hb, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        ho = hb.copy()
        oo = Oracle(ho, prm)
        oo.residual_core(RES_FLOW | RES_TURB)
        want = oo.wall_forces(ref_point, p_ref)
        got[name] = _device_forces(prm, hb, ref_point, p_ref)
        scale = np.abs(want).max(axis=1, keepdims=True)
        assert (scale > 0).all(), name
        assert (np.abs(got[name] - want) <= 1e-11 * scale).all(), (name, (got[name] - want) / scale)
    scale = np.abs(got["o_grid"]).max(axis=1, keepdims=True)
    for name in ("o_grid_jk", "o_grid_ki"):     # the same cylinder, the wall normal along j and along i
        assert (np.abs(got[name] - got["o_grid"]) <= 1e-12 * scale).all(), (name, (got[name] - got["o_grid"]) / scale)


# ---------------------------------------------------------------------------------------------------------------------
# equivariance of the device under the axis permutation (DADI and residual averaging sweep in a fixed order: left out)
@pytest.mark.parametrize("disc", list(DISCS))
@pytest.mark.parametrize("base", ["o_grid", "polar"])
def test_device_equivariance(cuda_lib, disc, base):
    prm = make_params({"equationType": "RANS", "discretization": DISCS[disc]})
    hb = meshes.o_grid(10, 12, 8, prm) if base == "o_grid" else meshes.polar_grid(10, 12, 8, prm)
    ow = hb.d.owned()

    def run(h):
        s = ADFLOW_B200(prm)
        try:
            s.addBlock(h)
            s.residual(RES_FLOW | RES_TURB | RES_SKIP_PREAMBLE)
            dw = s.downloadResidual(0)
            s.timeStep(False)
            dtl = np.zeros(h.d.box)
            dtl[1:h.d.ie + 1, 1:h.d.je + 1, 1:h.d.ke + 1] = s.downloadIntermed(0)["dtl"]
            return dw, dtl
        finally:
            s.close()

    dw0, dtl0 = run(hb)
    for perm in meshes.CYCLIC[1:]:
        dw, dtl = run(meshes.permute_axes(hb, perm))
        dw, dtl = meshes.unpermute(dw, perm), meshes.unpermute(dtl, perm)
        for l in range(hb.nw):
            e = rel_max(dw[ow + (l,)], dw0[ow + (l,)])
            assert e <= 10 * ORACLE_EQUIVARIANCE_DW, (perm, l, e)
        e = rel_max(dtl[ow], dtl0[ow])
        assert e <= 10 * ORACLE_EQUIVARIANCE_DTL, (perm, e)


# ---------------------------------------------------------------------------------------------------------------------
# a 3W multigrid cycle on the O-grid, the periodic lists on every level (both halo layers on the finest, the first halos
# on the coarse levels)
def _oracle_mg_cycle(prm, levels, pats, cycling, dadi_subiter):
    """executeMGCycle (tests/test_mg_gpu.py: oracle_mg_cycle) with the exchange of each level's own pattern where the
    smoothers and the grid transfers call whalo1: after every RK stage and DADI step, after the restriction's BCs on the
    coarse level, after the prolongation's BCs on the fine level"""
    from adflow_b200.halo import comm_vars
    from test_mg_gpu import oracle_transfer_to_coarse

    vars_ = lambda hb: comm_vars(hb, 1, 5, True, True, prm.equations != 1, False)  # noqa: E731

    def xch(lv):
        exchange_numpy([levels[lv]], pats[lv], vars_)

    def smooth(lv):
        o = Oracle(levels[lv], prm)
        if dadi_subiter:
            for q in range(dadi_subiter):
                o.dadi_step(); xch(lv)
                if q < dadi_subiter - 1:
                    o.residual_block(1.0)
            return
        np.copyto(o.hb.wn, o.hb.w[..., :5]); np.copyto(o.hb.pn, o.hb.p)
        for st in range(1, prm.nRKStages + 1):
            o.rk_stage(st); xch(lv)
            if st < prm.nRKStages:
                o.residual_block(prm.cdisRK[st])

    lv = 0
    for n, c in enumerate(cycling):
        if c == -1:
            lv -= 1
            Oracle(levels[lv], prm).mg_prolong(Oracle(levels[lv + 1], prm))
            Oracle(levels[lv], prm).apply_flow_bc(lv == 0); xch(lv)
        elif c == 0:
            if n > 0 and cycling[n - 1] != 1:
                o = Oracle(levels[lv], prm)
                o.time_step(True); o.residual_block(prm.cdisRK[0])
            smooth(lv)
        else:
            f, co = levels[lv], levels[lv + 1]
            of, oc = Oracle(f, prm), Oracle(co, prm)
            of.time_step(False); of.residual_block(prm.cdisRK[0])
            oc.mg_restrict(of); oc.apply_flow_bc(False); xch(lv + 1)
            oc.time_step(True); oc.mg_store_w1(); oc.residual_block_coarse(prm.cdisRK[0], init=0); oc.mg_forcing()
            lv += 1
    o = Oracle(levels[0], prm)
    o.time_step(True); o.residual_block(prm.cdisRK[0])


# Far field on both i faces: the default symmetry plane at x = 0 stands across the free stream, and the stagnation
# transient it starts changes rho by 0.7 of its size over one 3W RK cycle and makes the oracle's 3W DADI cycle overflow at
# the default CFL; with far field the cycle moves rho by 5 to 7 % of its size.
@pytest.mark.parametrize("eq,smoother", [("laminar NS", "RK"), ("Euler", "RK"), ("Euler", "DADI"), ("laminar NS", "DADI")])
def test_mg_3w_cycle_with_the_cut_on_every_level(cuda_lib, eq, smoother):
    from adflow_b200 import synthetic as syn

    prm, fine, _ = block("o_grid", eq, {"nRKStages": 3, "resAveraging": "never",
                                        "smoother": "DADI" if smoother == "DADI" else "Runge-Kutta"}, shape=(10, 12, 8),
                         i_faces=(syn.BC_FARFIELD, syn.BC_FARFIELD))
    levels = [fine]
    for _ in range(2):
        levels.append(meshes.coarse_level(levels[-1], prm))
    assert levels[-1].d.ny == 3
    pats = [meshes.self_periodic_pattern(h, 2 if q == 0 else 1) for q, h in enumerate(levels)]
    o = Oracle(fine, prm)
    o.apply_flow_bc(True)
    exchange_numpy([fine], pats[0], meshes.state_vars)
    dev = [h.copy() for h in levels]
    o.time_step(True); fine.fw[...] = 0; o.residual_block(prm.cdisRK[0])
    w0 = fine.w.copy()
    cyc = ADFLOW_B200.cycleStrategy("3w")
    sub = 2 if smoother == "DADI" else 0
    _oracle_mg_cycle(prm, levels, pats, cyc, sub)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(dev[0])
        for q in (1, 2):
            s.addCoarseBlock(dev[q], q - 1)
        for q in range(3):
            s.setCommPattern(pats[q], level=q + 1, block_offset=q)
        s.timeStep(False)
        s.smootherResidual(0)
        if sub:
            s.mgCycle(cyc, smoother="DADI", n_subiterations=sub)
        else:
            s.mgCycle(cyc)
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = fine.d.owned()
    tol_change, tol_w = (1e-7, 1e-9) if sub else (1e-8, 1e-10)
    for l in range(5):
        a, b = w[ow + (l,)] - w0[ow + (l,)], fine.w[ow + (l,)] - w0[ow + (l,)]
        assert np.abs(b).max() > 0
        assert rel_l2(a, b) < tol_change, ("state change over the cycle", l, rel_l2(a, b))
        if not sub:
            assert rel_l2(dw[ow + (l,)], fine.dw[ow + (l,)]) < 1e-8, ("residual after the cycle", l)
    assert rel_max(w[..., :5], fine.w[..., :5]) < tol_w    # halos incl. the exchanged ones
    assert np.abs(fine.w[ow + (0,)] - w0[ow + (0,)]).max() < 0.1 * np.abs(w0[ow + (0,)]).max()


# ---------------------------------------------------------------------------------------------------------------------
# convergence monitor: sums and maxima of adfb_monitor against the restatement of test_monitor_gpu.py, after a full
# residual with the cut's exchange
@pytest.mark.parametrize("name,eq", BLOCKS, ids=IDS)
def test_monitor(cuda_lib, name, eq):
    import monitor_ref as MR
    from test_monitor_gpu import _check, _host_blocks

    prm, hb, pat = block(name, eq)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.setCommPattern(pat)
        s.residual(flags_of(prm))
        host = _host_blocks(s, [0])
        for what in (1, 2, 3):
            got = s.monitorSums(1, what)
            _check(got, MR.monitor_sums(host, prm, what), what)
        full = MR.monitor_sums(host, prm)
        assert full[6] > 0 and full[8] > 0 and (eq != "RANS" or full[9] > 0)
    finally:
        s.close()
