"""The vector entry points on several blocks of different shapes per device: state / residual vectors, FormFunction_mf (one
shot and slab pipeline), the MFFD products, the ANK pieces, device GMRES, residual norms and wall forces, and the smoothers.

A rank of the reference owns several blocks, and every vector of the NK / ANK solvers is the concatenation of the local
level-1 blocks in block-id order; the library writes the per-block offsets of that concatenation by hand, once per entry
point.  The blocks of the set below have no exchange partners, so the multi-block result must equal the per-block oracle
results, concatenated.  The shapes differ (even and odd NI, different k-chunk counts, one block too short for the slab
pipeline), the walls sit on five different faces, one block has faces split into 14 pieces, and a level-2 block sits
between level-1 block ids: every offset loop has to skip it.  The element that decides a reduction sits in the last
level-1 block, so an offset or length that drops or shifts the tail changes the answer."""
import ctypes as C

import numpy as np
import pytest

from adflow_b200 import make_params
from adflow_b200 import synthetic as syn
from adflow_b200.halo import BlockGrid, build_cartesian_pattern, make_grid_blocks
from adflow_b200.params import make_ank_params
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_SKIP_PREAMBLE, RES_STORE_WALL, RES_TURB
from oracle.pyoracle import Oracle

from test_ank_gpu import _host_gmres, oracle_ank_function, oracle_blocks, vec_of
from test_halo_gpu import oracle_multiblock_residual
from util import FLOW, MIXED, TURB, oracle_form_function, rel_l2, rel_max, split_faces

pytestmark = pytest.mark.gpu

IMIN, IMAX, JMIN, JMAX, KMIN, KMAX = 1, 2, 3, 4, 5, 6
SYMM, WALL, FAR, ISOWALL = 1, 2, 3, 6
VISCOUS_FIRST = lambda s_: 0 if s_["bcType"] in (WALL, ISOWALL) else 1  # noqa: E731  (the reference numbers walls first)


def state_vec(hb):
    return np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()


def pinned(n):
    import torch

    return torch.empty(n, dtype=torch.float64).pin_memory()


class BlockSet:
    """Independent synthetic blocks, each with its own seed, registered in the order of `names`:
    A 24 x 16 x 32, default faces: even NI (TMA tiles), 8 k chunks (a 4-slab pipeline at the default 6 slabs);
    coarse: the level-2 block of A (addCoarseBlock), registered right after A;
    B 17 x 13 x 20, walls on IMAX (isothermal) and JMIN: odd NI (cp.async tiles), 5 chunks (a 2-slab pipeline);
    C 12 x 9 x 18, faces split by util.MIXED: 14 subfaces (no device subface list), wall pieces on KMIN, IMIN and JMAX;
    D 6 x 5 x 7: nz < 16, the slab pipeline does not apply while it is registered."""

    SHAPES = {"A": (24, 16, 32), "B": (17, 13, 20), "C": (12, 9, 18), "D": (6, 5, 7)}
    SEEDS = {"A": 1101, "B": 2203, "C": 3307, "D": 4409}

    def __init__(self, options=None, names=("A", "coarse", "B", "C", "D")):
        self.prm = prm = make_params(options)
        self.names = list(names)
        self.by_name = {}
        for n in self.names:
            if n == "coarse":
                continue
            kw = {}
            if n == "B":
                kw["physical_faces"] = {IMIN: FAR, IMAX: ISOWALL, JMIN: WALL, JMAX: FAR, KMIN: SYMM, KMAX: FAR}
            hb = syn.make_block(*self.SHAPES[n], prm, seed=self.SEEDS[n], **kw)
            if n == "C":
                split_faces(hb, prm, MIXED)
            hb.subfaces.sort(key=VISCOUS_FIRST)
            self.by_name[n] = hb
        self.coarse = syn.make_coarse_block(self.by_name["A"], prm) if "coarse" in self.names else None
        self.blocks = [self.by_name[n] for n in self.names if n != "coarse"]   # level 1, in device block-id order

    def register(self, s):
        """device ids in the order of `names`; returns the level-1 ids"""
        ids = []
        for n in self.names:
            if n == "coarse":
                s.addCoarseBlock(self.coarse, ids[self.names.index("A")] if "A" in self.names else 0)
            else:
                ids.append(s.addBlock(self.by_name[n]))
        return ids

    def parts(self, vec, per_cell):
        """views of a concatenated vector, one per level-1 block (per_cell entries per owned cell)"""
        out, off = [], 0
        for hb in self.blocks:
            n = hb.d.nx * hb.d.ny * hb.d.nz * per_cell
            out.append(vec[off:off + n])
            off += n
        assert off == len(vec)
        return out

    def concat(self, fn, *vecs, per_cell=None):
        """fn(hb, *slices of vecs) of every level-1 block, concatenated in block-id order"""
        per_cell = self.blocks[0].nw if per_cell is None else per_cell
        sl = [self.parts(v, per_cell) for v in vecs]
        return np.concatenate([np.asarray(fn(hb, *[p[q] for p in sl])).reshape(-1) for q, hb in enumerate(self.blocks)])

    def last_slice(self, per_cell):
        n = sum(hb.d.nx * hb.d.ny * hb.d.nz for hb in self.blocks[:-1]) * per_cell
        return slice(n, None)


def oracle_residual_vec(prm, hb):
    """getRes of the state in hb: blocketteRes (p / rlv / rev, BCs, owned rhoE, core) and dw / volRef"""
    d = hb.d
    ow = d.owned()
    h2 = hb.copy()
    o = Oracle(h2, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(FLOW | TURB)
    return np.transpose(h2.dw[ow] / h2.volRef[ow][..., None], (2, 1, 0, 3)).reshape(-1)


# ---------------------------------------------------------------------------------------------------------------------
# 1. vector layout
def test_state_and_residual_vectors(cuda_lib):
    bs = BlockSet()
    U = bs.concat(lambda hb: state_vec(hb))
    s = ADFLOW_B200(bs.prm)
    try:
        ids = bs.register(s)
        assert s.getStateSize() == U.size
        assert np.array_equal(s.getStates(), U)
        # setStates: each block its own slice of the owned cells, halos untouched
        before = [s.downloadState(q)[0] for q in ids]
        U2 = U * (1.0 + 0.01 * np.random.default_rng(8).standard_normal(U.size))
        s.setStates(U2)
        for q, hb, v, w0 in zip(ids, bs.blocks, bs.parts(U2, 6), before):
            w = s.downloadState(q)[0]
            ow = hb.d.owned()
            assert np.array_equal(w[ow], v.reshape(hb.d.nz, hb.d.ny, hb.d.nx, hb.nw).transpose(2, 1, 0, 3)), q
            halo = np.ones(hb.d.box, bool)
            halo[ow] = False
            assert np.array_equal(w[halo], w0[halo]), q
        assert np.array_equal(s.getStates(), U2)
        s.setStates(U)
        r = s.getResidual()
    finally:
        s.close()
    want = bs.concat(lambda hb: oracle_residual_vec(bs.prm, hb))
    assert rel_l2(r, want) < 1e-12, rel_l2(r, want)


# ---------------------------------------------------------------------------------------------------------------------
# 2. form function: one shot and slab pipeline
@pytest.mark.parametrize("options", [None, {"equationType": "Euler"}], ids=["RANS", "Euler"])
def test_form_function_and_pipeline(cuda_lib, monkeypatch, options):
    bs = BlockSet(options, names=("A", "coarse", "B", "C"))
    prm = bs.prm
    U = bs.concat(lambda hb: state_vec(hb))
    U = U * (1.0 + 1e-3 * np.random.default_rng(3).standard_normal(U.size))
    if prm.equations == syn.RANS:
        U[bs.last_slice(6)][5::6][:9] = -1.0        # setW's turbulence clip in the last block
    r_orc = bs.concat(lambda hb, u: oracle_form_function(prm, hb, u), U)
    n = U.size
    runs = {}
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        assert s.getStateSize() == n
        r_page = s.formFunction(U)
        hw, hr = pinned(n), pinned(n)
        hw.numpy()[:] = U
        for slabs in ("0", "3", "6"):
            monkeypatch.setenv("ADFB_FF_PIPE", slabs)
            hr.numpy()[:] = np.nan
            s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)     # first call captures the graph
            hr.numpy()[:] = np.nan
            c0 = s.launchCount()
            s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
            runs[slabs] = (hr.numpy().copy(), s.launchCount() - c0)
    finally:
        s.close()
    assert rel_l2(r_page, r_orc) < 1e-12, rel_l2(r_page, r_orc)
    r_one = runs["0"][0]
    assert np.array_equal(r_one, r_page)
    scale = np.abs(r_one).max()
    for slabs in ("3", "6"):
        r_pipe, nl = runs[slabs]
        assert np.isfinite(r_pipe).all()
        assert np.abs(r_pipe - r_one).max() <= 1e-13 * scale, (slabs, np.abs(r_pipe - r_one).max() / scale)
        assert rel_l2(r_pipe, r_orc) < 1e-11
        assert nl != runs["0"][1], slabs                # the pipeline ran: another launch sequence than the one shot
    assert runs["3"][1] != runs["6"][1]                # A is cut into 3 slabs, then 4
    assert rel_l2(r_one, r_orc) < 1e-11


def test_form_function_pipeline_refused_for_a_short_block(cuda_lib, monkeypatch):
    """with D (nz < 16) registered the page-locked call takes the one-shot path: same launches, same bits as pageable"""
    bs = BlockSet()
    prm = bs.prm
    U = bs.concat(lambda hb: state_vec(hb))
    U = U * (1.0 + 1e-3 * np.random.default_rng(4).standard_normal(U.size))
    n = U.size
    monkeypatch.delenv("ADFB_FF_PIPE", raising=False)
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        r_page = s.formFunction(U)
        c0 = s.launchCount()
        r_page2 = s.formFunction(U)
        n_page = s.launchCount() - c0
        hw, hr = pinned(n), pinned(n)
        hw.numpy()[:] = U
        hr.numpy()[:] = np.nan
        c0 = s.launchCount()
        s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        n_pin = s.launchCount() - c0
        r_pin = hr.numpy().copy()
    finally:
        s.close()
    assert np.array_equal(r_page, r_page2)
    assert np.array_equal(r_pin, r_page)
    assert n_pin == n_page
    r_orc = bs.concat(lambda hb, u: oracle_form_function(prm, hb, u), U)
    assert rel_l2(r_page, r_orc) < 1e-12


# ---------------------------------------------------------------------------------------------------------------------
# 3. MFFD products
def test_mffd_products(cuda_lib, monkeypatch):
    import torch

    bs = BlockSet()
    prm = bs.prm
    U = bs.concat(lambda hb: state_vec(hb))
    rng = np.random.default_rng(314)
    a = rng.standard_normal(U.size) * np.abs(U).clip(1e-6)
    a[bs.last_slice(6)] *= 10.0        # the tail dominates ||a||
    h = 1e-6
    monkeypatch.delenv("ADFB_MFFD_FUSED", raising=False)
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        s.mffdSetBase(U)
        y = s.mffdApply(a, h)
        assert s.mffdLastH() == h
        y_wp = s.mffdApply(a, -1.0)
        h_wp = s.mffdLastH()
        # device-resident vectors: the same bits
        y_host = s.mffdApply(a, 1e-7)
        da = torch.from_numpy(a).cuda()
        dy = torch.zeros_like(da)
        s.mffdApplyDevice(da.data_ptr(), dy.data_ptr(), da.numel(), 1e-7)
        y_dev = dy.cpu().numpy()
        # fused perturbation / difference quotient: every block takes the tile kernel, its epilogue writes rows at cell0
        y0 = s.mffdApply(a, 3e-7).copy()
        monkeypatch.setenv("ADFB_MFFD_FUSED", "1")
        y1 = s.mffdApply(a, 1e-7).copy()
        y2 = s.mffdApply(a, 3e-7).copy()
        monkeypatch.delenv("ADFB_MFFD_FUSED")
    finally:
        s.close()
    F0 = bs.concat(lambda hb, u: oracle_form_function(prm, hb, u), U)
    F1 = bs.concat(lambda hb, u: oracle_form_function(prm, hb, u), U + h * a)
    yref = (F1 - F0) / h
    assert rel_l2(y, yref) < 1e-6, rel_l2(y, yref)
    hexp = np.sqrt(np.finfo(float).eps) * np.sqrt(1.0 + np.linalg.norm(U)) / np.linalg.norm(a)
    assert abs(h_wp - hexp) < 1e-12 * hexp, (h_wp, hexp)
    assert np.isfinite(y_wp).all()
    assert np.array_equal(y_dev, y_host)
    assert np.abs(y1).max() > 0
    assert np.array_equal(y1, y_host)
    assert np.array_equal(y2, y0) and not np.array_equal(y1, y2)


# ---------------------------------------------------------------------------------------------------------------------
# 4. ANK
def ank_oracle_setup(prm, ank, bs):
    """BCs, time step, speed of sound and shock sensor of every block (in place, so the device gets the same state);
    returns the concatenated time-step matrix"""
    Ts = []
    for hb in bs.blocks:
        o = Oracle(hb, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        o.time_step(True)
        o.call("orc_speed_of_sound", C.byref(prm))
        o.reference_shock_sensor()
        Ts.append(oracle_blocks(prm, ank, hb))
    return Ts


@pytest.mark.parametrize("coupled,kind", [(True, "VLR"), (False, "Turkel")])
def test_ank_operator_and_product(cuda_lib, coupled, kind):
    bs = BlockSet()
    prm = bs.prm
    ank = make_ank_params(cfl=5.0, coupled=coupled, char_time_step=kind, mach=0.8, cflLimit=50.0, turbCFLScale=2.0)
    ns = 6 if coupled else 5
    Ts = ank_oracle_setup(prm, ank, bs)
    U = bs.concat(lambda hb: vec_of(hb, ns), per_cell=ns)
    rng = np.random.default_rng(5)
    v = U * (1.0 + 0.01 * rng.standard_normal(U.size))
    a = rng.standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-6
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        s.ankSetParams(ank)
        assert s.ankVecSize() == U.size
        s.referenceShockSensor()
        s.residual(RES_FLOW | RES_TURB | 4)
        s.ankTimeStepMat()
        F = s.ankFormFunction(v)
        s.ankMffdSetBase(U)
        y = s.ankMffdApply(a, h)
    finally:
        s.close()
    Tq = {id(hb): T for hb, T in zip(bs.blocks, Ts)}
    fn = lambda hb, x: oracle_ank_function(prm, ank, hb, Tq[id(hb)], x)  # noqa: E731
    Fref = bs.concat(fn, v, per_cell=ns)
    yref = (bs.concat(fn, U + h * a, per_cell=ns) - bs.concat(fn, U, per_cell=ns)) / h
    assert rel_l2(F, Fref) < 1e-11, rel_l2(F, Fref)
    assert rel_l2(y, yref) < 1e-5, rel_l2(y, yref)
    # the time-step term of the last block is really there
    T_last, v_last = Ts[-1], bs.parts(v, ns)[-1]
    assert np.abs(np.einsum("qlm,qm->ql", T_last, v_last.reshape(-1, ns))).max() > 0


@pytest.mark.parametrize("coupled", [False, True])
def test_ank_physicality_check(cuda_lib, coupled):
    bs = BlockSet()
    prm = bs.prm
    ank = make_ank_params(coupled=coupled)
    ns = 6 if coupled else 5
    wv = bs.concat(lambda hb: vec_of(hb, ns), per_cell=ns)
    rng = np.random.default_rng(11)
    dv = rng.standard_normal(wv.size) * np.abs(wv) * 0.4
    # the step that decides lambda sits in the last block: a density drop of 5 rho in one cell (and clipped SA updates)
    tail = bs.last_slice(ns)
    dv[tail][ns * 17] = -5.0 * wv[tail][ns * 17]
    if coupled:
        dv[tail][5::6][:40] = wv[tail][5::6][:40] * 500.0
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        s.ankSetParams(ank)
        for lam0 in (1.0, 0.03):
            per_block, d_ref = [], []
            for hb, w_q, d_q in zip(bs.blocks, bs.parts(wv, ns), bs.parts(dv, ns)):
                dq = d_q.copy()
                per_block.append(Oracle(hb, prm).ank_physicality_check(ank, w_q.copy(), dq, lam0))
                d_ref.append(dq)
            lam_ref, d_ref = min(per_block), np.concatenate(d_ref)
            if lam0 == 1.0:
                assert per_block[-1] < min(per_block[:-1])
            lam, d_dev = s.ankPhysicalityCheck(wv, dv, lam0)
            assert lam == lam_ref and 0 < lam <= lam0, (lam, lam_ref)
            assert np.array_equal(d_dev, d_ref)
    finally:
        s.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5. turbulence KSP of the decoupled ANK
def oracle_turb_function(prm, ank, hb, v):
    """FormFunction_mf_turb of one block (test_ank_gpu.test_turbulence_ksp_pieces)"""
    ow = hb.d.owned()
    h2 = hb.copy()
    o = Oracle(h2, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    dtl = h2.dtl.copy()
    h2.w[ow + (5,)] = np.transpose(np.asarray(v).reshape(hb.d.nz, hb.d.ny, hb.d.nx), (2, 1, 0))
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, hb.d.il, 2, hb.d.jl, 2, hb.d.kl)
    o.residual_core(TURB)
    h2.dtl[...] = dtl
    v = np.ascontiguousarray(v)
    r = np.empty_like(v)
    o.L.orc_ank_turb_rvec(C.byref(o.ob), C.byref(prm), C.byref(ank), v.ctypes.data_as(C.c_void_p), r.ctypes.data_as(C.c_void_p))
    return r


def test_turbulence_ksp_pieces(cuda_lib):
    bs = BlockSet()
    prm = bs.prm
    ank = make_ank_params(cfl=5.0, coupled=False, physLSTolTurb=0.99, stepMin=0.01, stepFactor=1.0)
    U = bs.concat(lambda hb: np.transpose(hb.w[hb.d.owned()][..., 5], (2, 1, 0)).reshape(-1), per_cell=1)
    rng = np.random.default_rng(5)
    vin = U * (1.0 + 0.01 * rng.standard_normal(U.size))
    a = rng.standard_normal(U.size) * np.abs(U)
    h = 1e-6
    dv = rng.standard_normal(U.size) * np.abs(U) * 0.4
    tail = bs.last_slice(1)
    dv[tail][:30] = U[tail][:30] * 500.0         # clipped updates (ratio below stepMin), in the last block
    dv[tail][40] = U[tail][40] * 20.0            # the update that decides lambda, in the last block
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        s.ankSetParams(ank)
        s.residual(FLOW | TURB | 4)
        r = s.ankFormFunctionTurb(vin)
        s.ankMffdTurbSetBase(U)
        y = s.ankMffdTurbApply(a, h)
        lam, dclip = s.ankPhysicalityCheckTurb(U, dv, 1.0)
    finally:
        s.close()
    fn = lambda hb, x: oracle_turb_function(prm, ank, hb, x)  # noqa: E731
    want = bs.concat(fn, vin, per_cell=1)
    assert rel_l2(r, want) < 1e-11, rel_l2(r, want)
    yref = (bs.concat(fn, U + h * a, per_cell=1) - bs.concat(fn, U, per_cell=1)) / h
    assert rel_l2(y, yref) < 1e-6, rel_l2(y, yref)
    f = Oracle(bs.blocks[0], prm).L.orc_ank_physicality_check_turb
    f.restype = C.c_double
    lams, d_ref = [], []
    for u_q, d_q in zip(bs.parts(U, 1), bs.parts(dv, 1)):
        u_q, dq = np.ascontiguousarray(u_q), d_q.copy()
        lams.append(f(C.byref(ank), C.c_long(u_q.size), u_q.ctypes.data_as(C.c_void_p), dq.ctypes.data_as(C.c_void_p), C.c_double(1.0)))
        d_ref.append(dq)
    d_ref = np.concatenate(d_ref)
    assert lams[-1] < min(lams[:-1])
    assert lam == min(lams), (lam, lams)
    assert np.array_equal(dclip, d_ref) and np.abs(d_ref - dv).max() > 0


# ---------------------------------------------------------------------------------------------------------------------
# 6. device GMRES
def test_device_gmres_on_the_block_diagonal_time_step_matrix(cuda_lib):
    """op TSMAT over all blocks: two restart cycles reproduce a host GMRES, the recurrence's estimate is the true residual,
    and with the exact inverse as right preconditioner it converges at once"""
    import torch

    bs = BlockSet()
    prm = bs.prm
    ank = make_ank_params(cfl=3.0, coupled=True, char_time_step="VLR", cflLimit=20.0, turbCFLScale=2.0)
    ns = 6
    T = np.concatenate(ank_oracle_setup(prm, ank, bs))
    apply = lambda v: np.einsum("qlm,qm->ql", T, v.reshape(-1, ns)).reshape(-1)  # noqa: E731
    b = np.random.default_rng(2).standard_normal(T.shape[0] * ns)
    rtol, restart, max_its = 1e-12, 12, 24

    class DevVec:
        def __init__(self, ptr, n):
            self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 2}

    Tinv = torch.linalg.inv(torch.from_numpy(T).cuda())
    calls = []

    def pc(ctx, in_ptr, out_ptr, n):
        v = torch.as_tensor(DevVec(in_ptr, n), device="cuda").reshape(-1, ns)
        out = torch.as_tensor(DevVec(out_ptr, n), device="cuda").reshape(-1, ns)
        out.copy_(torch.einsum("qlm,qm->ql", Tinv, v))
        torch.cuda.synchronize()
        calls.append(n)
        return 0

    pc_c = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong)(pc)
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        s.ankSetParams(ank)
        s.residual(RES_FLOW | RES_TURB | 4)
        s.ankTimeStepMat()
        x, its, rn = s.gmresSolve(b, op="TSMAT", restart=restart, max_its=max_its, rtol=rtol)
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
    assert abs(rn / np.linalg.norm(b) - res) < 1e-6 * res + 1e-12
    assert res < 1.0
    assert np.linalg.norm(x - xh) < 1e-7 * np.linalg.norm(xh), np.linalg.norm(x - xh) / np.linalg.norm(xh)
    assert itp.value <= 2 and len(calls) >= 2
    assert np.linalg.norm(b - apply(xp)) < 1e-8 * np.linalg.norm(b)


def test_device_gmres_on_the_nk_product(cuda_lib):
    """op NK over all blocks against a host GMRES that applies the same device operator vector by vector"""
    bs = BlockSet()
    s = ADFLOW_B200(bs.prm)
    try:
        bs.register(s)
        s.applyBCs(True, True)
        U = s.getStates()
        s.mffdSetBase(U)
        apply = lambda v: s.mffdApply(v, -1.0)  # noqa: E731
        rtol, restart, max_its = 1e-3, 10, 10
        b = apply(np.random.default_rng(3).standard_normal(U.size) * np.abs(U).clip(1e-6) * 1e-3)
        x, its, rn = s.gmresSolve(b, op="NK", restart=restart, max_its=max_its, rtol=rtol)
        xh, its_h = _host_gmres(apply, b, restart, max_its, rtol)
    finally:
        s.close()
    assert np.isfinite(x).all() and its >= 1 and abs(its - its_h) <= 1
    assert rn <= np.linalg.norm(b) * (1 + 1e-12)
    assert np.linalg.norm(x - xh) < 2e-2 * np.linalg.norm(xh), np.linalg.norm(x - xh) / np.linalg.norm(xh)


# ---------------------------------------------------------------------------------------------------------------------
# 7. residual norms and wall forces
def test_residual_norms_and_wall_forces(cuda_lib):
    """walls on five faces of three blocks, two of them split into pieces (C: two wall pieces on KMIN)"""
    bs = BlockSet()
    prm = bs.prm
    ref_point, p_ref = (0.3, -0.2, 0.1), 2.5
    want_n, want_f, nwall = np.zeros(2), np.zeros((4, 3)), 0
    for hb in bs.blocks:
        o = Oracle(hb, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)      # halos consistent on both sides
        ho = hb.copy()
        oo = Oracle(ho, prm)
        oo.residual_core(RES_FLOW | RES_TURB)
        want_n += oo.norms()
        want_f += oo.wall_forces(ref_point, p_ref)
        nwall += sum(s_["bcType"] in (WALL, ISOWALL) for s_ in hb.subfaces)
    assert nwall == 8
    s = ADFLOW_B200(prm)
    try:
        bs.register(s)
        s.residual(RES_FLOW | RES_TURB | RES_STORE_WALL | RES_SKIP_PREAMBLE)
        norms = s.getResNorms()
        got = s.getForces(ref_point, p_ref)
    finally:
        s.close()
    assert (np.abs(norms - want_n) <= 1e-11 * want_n).all(), (norms - want_n) / want_n
    scale = np.abs(want_f).max(axis=1, keepdims=True)
    assert (scale > 0).all()
    assert (np.abs(got - want_f) <= 1e-11 * scale).all(), (got - want_f) / scale


# ---------------------------------------------------------------------------------------------------------------------
# 8. smoothers on blocks of different shapes (residual averaging and SA lines pick a kernel per block shape)
def test_rk_cycle_on_blocks_of_different_shapes(cuda_lib):
    bs = BlockSet({"nRKStages": 5, "resAveraging": "alternate"}, names=("A", "B", "C"))
    prm = bs.prm
    refs = []
    for hb in bs.blocks:
        ho = hb.copy()
        o = Oracle(ho, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        o.time_step(True)
        ho.fw[...] = 0
        o.residual_block(prm.cdisRK[0])
        o.rk_smoother()
        refs.append(ho)
    s = ADFLOW_B200(prm)
    try:
        ids = bs.register(s)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        s.rkCycle()
        states = [s.downloadState(q) for q in ids]
    finally:
        s.close()
    for name, hb, ho, (w, p, rlv, rev) in zip(bs.names, bs.blocks, refs, states):
        ow = hb.d.owned()
        dwv, dwo = w[ow] - hb.w[ow], ho.w[ow] - hb.w[ow]
        assert np.abs(dwo[..., :5]).max() > 1e-8, name
        for l in range(5):
            assert rel_l2(dwv[..., l], dwo[..., l]) < 1e-10, (name, l, rel_l2(dwv[..., l], dwo[..., l]))
        assert rel_max(w[..., :5], ho.w[..., :5]) < 1e-11, name
        assert rel_max(p, ho.p) < 1e-11, name


def test_sa_ddadi_on_blocks_of_different_shapes(cuda_lib):
    niter = 2
    bs = BlockSet(names=("A", "B", "C"))
    prm = bs.prm
    refs = []
    for hb in bs.blocks:
        ho = hb.copy()
        o = Oracle(ho, prm)
        o.apply_turb_bc(True); o.apply_flow_bc(True)
        for _ in range(niter):
            o.sa_block()
        refs.append(ho)
    s = ADFLOW_B200(prm)
    try:
        ids = bs.register(s)
        s.applyBCs(True, True)
        s.turbSolveDDADI(niter)
        out = [(s.downloadState(q), s.downloadResidual(q)) for q in ids]
    finally:
        s.close()
    for name, hb, ho, ((w, p, rlv, rev), dw) in zip(bs.names, bs.blocks, refs, out):
        ow = hb.d.owned()
        assert rel_l2(dw[ow + (5,)], ho.dw[ow + (5,)]) < 1e-10, name
        dn, do = w[ow + (5,)] - hb.w[ow + (5,)], ho.w[ow + (5,)] - hb.w[ow + (5,)]
        assert np.abs(do).max() > 0, name
        assert rel_l2(dn, do) < 1e-9, (name, rel_l2(dn, do))
        assert rel_max(w[..., 5], ho.w[..., 5]) < 1e-10, name
        d = hb.d
        c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
        assert rel_max(rev[c1], ho.rev[c1]) < 1e-10, name


# ---------------------------------------------------------------------------------------------------------------------
# 9. blocks with exchange partners: the one-shot path with a 1-to-1 pattern
def test_form_function_and_product_with_an_exchange_pattern(cuda_lib, monkeypatch):
    """2 x 1 x 2 blocks of 9 x 8 x 18 joined by a 1-to-1 pattern.  The BCs run before the exchange, so the BC halos next to
    a block interface follow the interface halos of the PREVIOUS evaluation: the oracle keeps its blocks from one
    evaluation to the next, in the order the device evaluates."""
    prm = make_params()
    grid = BlockGrid((2, 1, 2), (9, 8, 18), nranks=1)
    blocks = make_grid_blocks(grid, 0, prm)
    pat = build_cartesian_pattern(grid, 0)
    ref = [b.copy() for b in blocks]

    def oracle_ff(vec):
        off = 0
        for hb in ref:
            d = hb.d
            n = d.nx * d.ny * d.nz * hb.nw
            v = vec[off:off + n].reshape(d.nz, d.ny, d.nx, hb.nw).transpose(2, 1, 0, 3).copy()
            v[..., 5] = np.maximum(1e-6 * prm.wInf[5], v[..., 5])      # setW's turbulence clip
            hb.w[d.owned()] = v
            off += n
        oracle_multiblock_residual(prm, grid, ref, pat)
        out = []
        for hb in ref:
            ow = hb.d.owned()
            r = hb.dw[ow] / hb.volRef[ow][..., None]
            r[..., 5] *= prm.turbResScale
            out.append(np.transpose(r, (2, 1, 0, 3)).reshape(-1))
        return np.concatenate(out)

    U = np.concatenate([state_vec(hb) for hb in blocks])
    U = U * (1.0 + 1e-3 * np.random.default_rng(6).standard_normal(U.size))
    rng = np.random.default_rng(314)
    a = rng.standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-6
    n = U.size
    monkeypatch.delenv("ADFB_FF_PIPE", raising=False)
    monkeypatch.delenv("ADFB_MFFD_FUSED", raising=False)
    s = ADFLOW_B200(prm)
    try:
        for hb in blocks:
            s.addBlock(hb)
        s.setCommPattern(pat)
        r1 = s.formFunction(U)
        r2 = s.formFunction(U)
        hw, hr = pinned(n), pinned(n)
        hw.numpy()[:] = U
        hr.numpy()[:] = np.nan
        s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        r_pin = hr.numpy().copy()
        s.mffdSetBase(U)
        y = s.mffdApply(a, h)
    finally:
        s.close()
    R1 = oracle_ff(U)
    R2 = oracle_ff(U)
    F0 = oracle_ff(U)           # mffdSetBase
    F1 = oracle_ff(U + h * a)
    assert rel_l2(r1, R1) < 1e-12, rel_l2(r1, R1)
    assert rel_l2(r2, R2) < 1e-12, rel_l2(r2, R2)
    assert np.array_equal(r_pin, r2)          # the pattern ties slabs together: the page-locked call is the one shot
    yref = (F1 - F0) / h
    assert rel_l2(y, yref) < 1e-6, rel_l2(y, yref)
