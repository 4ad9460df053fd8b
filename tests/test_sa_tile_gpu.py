"""The SA-row tile kernel k_sa (adflow_b200/csrc/sa_tile.cuh) in the launch configurations large blocks get.

On the small blocks of the rest of the GPU suite sa_tile_choose gives every CTA one k plane, so the carry from plane to
plane, the load of plane k+2 into the buffer plane k-1 left, the cp.async group accounting, the forming of nu in the
next buffer and the trailing barrier never run past the first plane.  ADFB_SA_TILE=TX,TY,kChunk forces a thread tile and
a k chunk; the configurations are those of tests/sa_configs.py, which the CPU emulation (tests/test_sa_emul.py) runs as
well.  Each is held against the oracle plane by plane, and its SA row and flow rows against a run with the chooser's own
configuration bit for bit: every cell runs the same expression sequence whatever the tile and chunk, and the two sums of
a shared face commute.

The variable is read at every launch, but a CUDA graph keeps the configuration it was captured with, so every run here
sets it before its context is created."""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import regimes as R
import sa_configs as SC
from adflow_b200.params import make_ank_params
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_SKIP_PREAMBLE, RES_TURB
from oracle.pyoracle import Oracle
from test_regimes_reach import assert_reaches
from util import MIXED, case, oracle_form_function, oracle_residual

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CORE = RES_FLOW | RES_TURB | RES_SKIP_PREAMBLE
SHAPE = SC.SHAPES[0]
CHUNKED = [(7, 4, 3), (16, 8, 5)]   # two chunked configurations for the options, regimes and entry points


def _tile_env(tile):
    return {"ADFB_SA_TILE": None if tile is None else "%d,%d,%d" % tuple(tile)}


class _env:
    """os.environ with some variables set (value) or removed (None) inside the block"""

    def __init__(self, **kv):
        self.kv = kv

    def __enter__(self):
        self.old = {k: os.environ.get(k) for k in self.kv}
        for k, v in self.kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v

    def __exit__(self, *a):
        for k, v in self.old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def _residual(prm, blocks, tile, flags=CORE):
    """dw of each block after one residual evaluation in a fresh context, the SA row formed with `tile` (None: the chooser)"""
    with _env(**_tile_env(tile)):
        s = ADFLOW_B200(prm)
        try:
            for hb in blocks:
                s.addBlock(hb)
            s.residual(flags)
            return [s.downloadResidual(n) for n in range(len(blocks))]
        finally:
            s.close()


def _same_rows(hb, got, want, what=""):
    ow = hb.d.owned()
    for l in range(hb.nw):
        assert np.array_equal(got[ow + (l,)], want[ow + (l,)]), "%s row %d differs from the chooser's configuration" % (what, l)


def _check(prm, hb, tiles, ref=None, flags=CORE):
    """each tile's SA row against the oracle plane by plane, and all rows bitwise against the chooser's configuration"""
    ow = hb.d.owned()
    if ref is None:
        ref = oracle_residual(prm, hb, RES_FLOW | RES_TURB).dw
    base = _residual(prm, [hb], None, flags)[0]
    SC.assert_sa_planes(base[ow + (5,)], ref[ow + (5,)], what="chooser")
    out = []
    for t in tiles:
        dw = _residual(prm, [hb], t, flags)[0]
        SC.assert_sa_planes(dw[ow + (5,)], ref[ow + (5,)], what="SA row %s" % (t,))
        _same_rows(hb, dw, base, str(t))
        out.append(dw)
    return out


# ---------------------------------------------------------------------------------------------------------------------
# a. configuration matrix
@pytest.fixture(scope="module")
def block(request, cuda_lib):
    """block, oracle residual and the residual with the chooser's configuration, formed in the set-up (outside the call
    the kernel trace records)"""
    shape = request.param
    prm, hb = case(*shape)
    ref = oracle_residual(prm, hb, RES_FLOW | RES_TURB).dw
    base = _residual(prm, [hb], None)[0]
    return prm, hb, ref, base


@pytest.mark.parametrize("block,tile", SC.CONFIGS, indirect=["block"], ids=[SC.config_id(c) for c in SC.CONFIGS])
def test_configuration_matrix(block, tile):
    prm, hb, ref, base = block
    dw = _residual(prm, [hb], tile)[0]
    ow = hb.d.owned()
    SC.assert_sa_planes(dw[ow + (5,)], ref[ow + (5,)])
    _same_rows(hb, dw, base)


def test_override_that_does_not_fit_is_not_launched(cuda_lib):
    """64 x 4 threads is more than SA_MAXT: the chooser's configuration runs (the launches are checked in the trace)"""
    prm, hb = case(*SHAPE)
    ref = oracle_residual(prm, hb, RES_FLOW | RES_TURB).dw
    dw = _residual(prm, [hb], (64, 4, 2))[0]
    ow = hb.d.owned()
    SC.assert_sa_planes(dw[ow + (5,)], ref[ow + (5,)])


def test_each_configuration_ran(cuda_lib, tmp_path):
    """the k_sa launches of the matrix, from the grid / block args of the Kineto trace (ADFB_NO_GRAPH=1: every launch is
    reported by itself): block TX * TY, grid (nx / TX, ny / TY, nPlanes / kChunk) rounded up; an override that does not
    fit launches as the chooser's pick"""
    import torch

    out = tmp_path / "launches.json"
    mod = os.path.join(HERE, "test_sa_tile_gpu.py")
    nodes = [mod + "::test_configuration_matrix", mod + "::test_override_that_does_not_fit_is_not_launched"]
    e = dict(os.environ, ADFB_NO_GRAPH="1")
    e.pop("ADFB_SA_TILE", None)
    e["PYTHONPATH"] = os.pathsep.join([HERE] + ([e["PYTHONPATH"]] if e.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-m", "pytest", "-p", "kernel_trace", "--kernel-launches", str(out), "-q", "-p", "no:cacheprovider",
                        "--rootdir", ROOT] + nodes, cwd=ROOT, env=e, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    with open(out) as f:
        seen = json.load(f)

    def k_sa(node):
        got = [(g, b) for n, g, b in seen[node] if n == "k_sa"]
        assert got, "%s: no k_sa launch in the trace" % node
        assert all(g is not None and b is not None for g, b in got), "the trace has no grid / block args"
        return {(tuple(g), tuple(b)) for g, b in got}

    for c in SC.CONFIGS:
        shape, tile = c
        node = [n for n in seen if n.endswith("test_configuration_matrix[%s]" % SC.config_id(c))]
        assert len(node) == 1, SC.config_id(c)
        assert k_sa(node[0]) == {SC.sa_grid(shape, shape[2], tile)}, SC.config_id(c)
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    pick = SC.sa_tile_choose(SHAPE, SHAPE[2], n_sm, SC.SA_CTAS_PER_SM)
    node = [n for n in seen if n.endswith("test_override_that_does_not_fit_is_not_launched")][0]
    assert k_sa(node) == {SC.sa_grid(SHAPE, SHAPE[2], pick)}


# ---------------------------------------------------------------------------------------------------------------------
# b. options, blanking, regimes
@pytest.mark.parametrize("opt", SC.OPTIONS, ids=lambda o: "-".join("%s=%s" % kv for kv in o.items()))
def test_options(cuda_lib, opt):
    prm, hb = case(*SHAPE, opt)
    _check(prm, hb, CHUNKED)


@pytest.mark.parametrize("tile", CHUNKED, ids=lambda t: "x".join(map(str, t)))
def test_blanked_cells_and_seam_planes(cuda_lib, tile):
    """iblank 0 and -1 scattered, and the whole first plane of the second chunk blanked (0) and the last plane of the
    first chunk a hole (-1): the rows there are zero, the carry across them is the unblanked one"""
    prm, hb = case(*SHAPE)
    ow = hb.d.owned()
    ib = hb.iblank[ow]
    ib[...] = np.random.default_rng(5).choice([1, 1, 1, 1, 0, -1], size=ib.shape)
    seam = tile[2]                      # owned plane index of the first plane of the second chunk
    ib[..., seam] = 0
    ib[..., seam - 1] = -1
    hb.iblank[ow] = ib
    dw = _check(prm, hb, [tile])[0]
    assert (dw[ow + (5,)][ib <= 0] == 0.0).all()


@pytest.mark.parametrize("regime,keys", [("low_reynolds", ["low_cell_re"]), ("stagnation", ["stagnant_j", "sa_rr_clip"])])
def test_regimes(cuda_lib, regime, keys):
    prm, hb = R.regime_case(regime, SHAPE)
    assert_reaches(prm, hb, regime, keys)
    _check(prm, hb, CHUNKED)


@pytest.mark.parametrize("seam", [0, 1])
@pytest.mark.parametrize("tile", CHUNKED, ids=lambda t: "x".join(map(str, t)))
def test_contact_on_a_chunk_seam(cuda_lib, tile, seam):
    """a density jump along k on the face where the second chunk starts, and one plane past it"""
    at = 2 + tile[2] + seam
    prm, hb = R.regime_case("contact_k", SHAPE, at=at)
    assert_reaches(prm, hb, "contact_k", ["sensor_cap_k"])
    _check(prm, hb, [tile])


# ---------------------------------------------------------------------------------------------------------------------
# c. entry points
def test_full_residual_with_preamble_and_split_faces(cuda_lib):
    """adfb_residual with the state preparation and BCs, every face in pieces (tests/util.py: MIXED)"""
    prm, hb = case(*SHAPE, split=MIXED)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(RES_FLOW | RES_TURB)
    _check(prm, hb, CHUNKED, ref=ho.dw, flags=RES_FLOW | RES_TURB)


def _rows(r, hb):
    """vector in (k, j, i, variable) order -> [row l as (i, j, k)]"""
    d = hb.d
    v = r.reshape(d.nz, d.ny, d.nx, hb.nw)
    return [np.transpose(v[..., l], (2, 1, 0)) for l in range(hb.nw)]


def _pinned(n):
    import torch

    return torch.empty(n, dtype=torch.float64).pin_memory()


def _form_function(prm, hb, U, tile, slabs):
    """(one-shot, pipelined with `slabs` slabs) form function in one context"""
    with _env(**_tile_env(tile)):
        s = ADFLOW_B200(prm)
        try:
            s.addBlock(hb)
            n = s.getStateSize()
            hw, hr = _pinned(n), _pinned(n)
            hw.numpy()[:] = U
            out = []
            for pipe in ("0", str(slabs)):
                hr.numpy()[:] = np.nan
                with _env(ADFB_FF_PIPE=pipe):
                    s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
                out.append(hr.numpy().copy())
            return out
        finally:
            s.close()


@pytest.mark.parametrize("slabs", [3, 6])
def test_pipelined_form_function(cuda_lib, slabs):
    """slabs of 4 .. 16 planes (multiples of the pipeline's 4-plane chunks): chunks of 3 and 5 planes cut every slab
    several times and none evenly"""
    prm, hb = case(21, 11, 48)
    U = np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()
    U = U * (1.0 + 1e-3 * np.random.default_rng(3).standard_normal(U.size))
    want = _rows(oracle_form_function(prm, hb, U), hb)
    one0, pipe0 = _form_function(prm, hb, U, None, slabs)
    for tile in CHUNKED:
        one, pipe = _form_function(prm, hb, U, tile, slabs)
        for r, r0, what in ((one, one0, "one-shot"), (pipe, pipe0, "pipelined")):
            got, got0 = _rows(r, hb), _rows(r0, hb)
            SC.assert_sa_planes(got[5], want[5], what="%s %s" % (what, tile))
            for l in range(6):
                assert np.array_equal(got[l], got0[l]), (what, tile, l)
        # the SA row does not depend on where the slabs cut it
        assert np.array_equal(_rows(pipe, hb)[5], _rows(one0, hb)[5]), tile


def test_fused_mffd_product(cuda_lib):
    """ADFB_MFFD_FUSED=1 (the difference quotient formed in k_sa's epilogue) is the three-pass product bit for bit, and
    neither depends on the configuration"""
    prm, hb = case(*SHAPE)
    U = np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()
    a = np.random.default_rng(2).standard_normal(U.size) * np.abs(U).clip(1e-6)
    ys = {}
    for tile in [None] + CHUNKED:
        for fused in ("0", "1"):
            with _env(ADFB_MFFD_FUSED=fused, **_tile_env(tile)):
                s = ADFLOW_B200(prm)
                try:
                    s.addBlock(hb)
                    s.mffdSetBase(U)
                    ys[tile, fused] = s.mffdApply(a, 1e-7).copy()
                finally:
                    s.close()
    y0 = ys[None, "0"]
    assert np.isfinite(y0).all() and np.abs(y0[5::6]).max() > 0
    for k, y in ys.items():
        assert np.array_equal(y, y0), k


def test_ank_turbulence_form_function(cuda_lib):
    """FormFunction_mf_turb of the decoupled ANK turbulence solve: the same bits in every configuration"""
    prm, hb = case(*SHAPE)
    ank = make_ank_params(cfl=5.0, coupled=False, physLSTolTurb=0.99, stepMin=0.01, stepFactor=1.0)
    U = np.ascontiguousarray(np.transpose(hb.w[hb.d.owned()][..., 5], (2, 1, 0)).reshape(-1))
    vin = U * (1.0 + 0.01 * np.random.default_rng(5).standard_normal(U.size))
    rs = []
    for tile in [None] + CHUNKED:
        with _env(**_tile_env(tile)):
            s = ADFLOW_B200(prm)
            try:
                s.addBlock(hb)
                s.ankSetParams(ank)
                s.residual(RES_FLOW | RES_TURB | 4)
                rs.append(s.ankFormFunctionTurb(vin).copy())
            finally:
                s.close()
    assert np.isfinite(rs[0]).all() and np.abs(rs[0]).max() > 0
    for r in rs[1:]:
        assert np.array_equal(r, rs[0])


def test_blocks_of_different_shapes_in_one_context(cuda_lib):
    """four blocks in one context: each gets the forced tile with the chunk clamped to its own planes"""
    shapes = [SC.SHAPES[0], SC.SHAPES[1], (12, 10, 4), (21, 6, 11)]
    prm = case(*shapes[0])[0]
    blocks = [case(*sh, seed=314 + n)[1] for n, sh in enumerate(shapes)]
    refs = [oracle_residual(prm, hb, RES_FLOW | RES_TURB).dw for hb in blocks]
    base = _residual(prm, blocks, None)
    for tile in CHUNKED:
        got = _residual(prm, blocks, tile)
        for hb, dw, dw0, ref in zip(blocks, got, base, refs):
            ow = hb.d.owned()
            SC.assert_sa_planes(dw[ow + (5,)], ref[ow + (5,)], what="block %s, %s" % (hb.d.nx, tile))
            _same_rows(hb, dw, dw0, str(tile))
