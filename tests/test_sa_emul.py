"""CPU emulation of the SA-row tile kernel k_sa (adflow_b200/csrc/sa_tile.cuh) against the oracle.

The kernel's per-thread phase functions are plain __host__ __device__ code; tests/emul/sa_emul.cu runs them thread by
thread with the shared-memory plane buffers in host memory (poisoned with NaN wherever nothing was loaded).  This checks
the tile logic (index maps, halos of one and two cells, k marching with carried faces, chunk seams and plane sub-ranges)
for several block and tile shapes without a GPU; the GPU suite checks the kernel itself."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import sa_configs as SC
from sa_configs import OPTIONS
from util import FLOW, TURB, case, oracle_residual, rel_l2, rel_max

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emul", "sa_emul.cu")
SO = os.path.join(HERE, "emul", "libsa_emul.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
TOL = 1e-12


def _build():
    deps = [SRC] + [os.path.join(HERE, "..", "adflow_b200", "csrc", f) for f in ("sa_tile.cuh", "adfb_common.cuh")]
    if os.path.exists(SO) and all(os.path.getmtime(SO) > os.path.getmtime(f) for f in deps):
        return SO
    if not (os.path.exists(NVCC) or shutil.which("nvcc")):
        pytest.skip("nvcc not available")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-o", SO, SRC])
    return SO


class SaEmulArrays(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w", "rlv", "si", "sj", "sk", "vol", "volRef", "d2Wall", "dw", "iblank")]


def run_emul(prm, hb, TX, TY, kc, n_sm=0, ctas=0, k_off=0, k_top=2 ** 31 - 1):
    """dw(itu1) by the emulated kernel (NaN outside the planes it forms); TX = 0: the host chooser's tile"""
    L = C.CDLL(_build())
    d = hb.d
    keep = {}
    ea = SaEmulArrays()
    for n in ("w", "rlv", "si", "sj", "sk", "vol", "volRef", "d2Wall", "iblank"):
        a = np.asfortranarray(getattr(hb, n))
        keep[n] = a
        setattr(ea, n, a.ctypes.data)
    dw = np.full(hb.dw.shape, np.nan, order="F")
    ea.dw = dw.ctypes.data
    L.emul_sa.argtypes = [C.c_int] * 3 + [C.c_void_p, C.c_void_p] + [C.c_int] * 7
    assert L.emul_sa(d.nx, d.ny, d.nz, C.byref(prm), C.byref(ea), TX, TY, kc, n_sm, ctas, k_off, k_top) == 0
    return dw[..., 5]


def _check(hb, got, want, planes=None):
    ow = hb.d.owned()
    a, b = got[ow], want[ow]
    if planes is not None:
        a, b = a[..., planes], b[..., planes]
    assert np.isfinite(a).all()
    assert rel_l2(a, b) < TOL and rel_max(a, b) < TOL, (rel_l2(a, b), rel_max(a, b))


@pytest.mark.parametrize("shape,tile", [((12, 10, 8), (32, 4, 3)), ((12, 10, 8), (16, 8, 8)), ((16, 9, 7), (7, 4, 3)),
                                         ((10, 6, 9), (5, 7, 1)), ((14, 8, 6), (3, 3, 2)), ((9, 11, 5), (10, 3, 4))])
def test_emulated_sa_row_matches_oracle(shape, tile):
    prm, hb = case(*shape)
    ho = oracle_residual(prm, hb, FLOW | TURB)
    _check(hb, run_emul(prm, hb, *tile), ho.dw[..., 5])


@pytest.mark.parametrize("opt", OPTIONS, ids=lambda o: "-".join("%s=%s" % kv for kv in o.items()))
@pytest.mark.parametrize("tile", [(7, 4, 3), (16, 8, 1)])
def test_emulated_sa_row_options(opt, tile):
    prm, hb = case(12, 10, 9, opt)
    ho = oracle_residual(prm, hb, FLOW | TURB)
    _check(hb, run_emul(prm, hb, *tile), ho.dw[..., 5])


def test_emulated_sa_row_iblank():
    """blanked (0) and hole (-1) cells get a zero row, on tile and chunk seams as well"""
    prm, hb = case(12, 10, 8)
    rng = np.random.default_rng(5)
    ow = hb.d.owned()
    ib = hb.iblank[ow]
    ib[...] = rng.choice([1, 1, 1, 0, -1], size=ib.shape)
    hb.iblank[ow] = ib
    ho = oracle_residual(prm, hb, FLOW | TURB)
    dw = run_emul(prm, hb, 5, 4, 3)
    _check(hb, dw, ho.dw[..., 5])
    assert (dw[ow][ib <= 0] == 0.0).all()


@pytest.mark.parametrize("k_off,k_top,kc", [(0, 5, 2), (3, 7, 1), (2, 9, 3), (5, 2 ** 31 - 1, 2)])
def test_emulated_sa_row_plane_ranges(k_off, k_top, kc):
    """the form-function pipeline's slabs: planes 2+kOff .. min(kl, kTop) only, nothing outside them is written"""
    prm, hb = case(11, 9, 10, {"turbulenceOrder": "second order"})
    ho = oracle_residual(prm, hb, FLOW | TURB)
    dw = run_emul(prm, hb, 7, 5, kc, k_off=k_off, k_top=k_top)
    kl = hb.d.kl
    hi = min(kl, k_top)
    sel = np.arange(2 + k_off, hi + 1) - 2      # owned-plane index
    _check(hb, dw, ho.dw[..., 5], planes=sel)
    rest = np.setdiff1d(np.arange(hb.d.nz), sel)
    assert np.isnan(dw[hb.d.owned()][..., rest]).all()


@pytest.mark.parametrize("shape,n_sm,ctas", [((96, 72, 64), 132, 4), ((24, 16, 12), 132, 4), ((20, 14, 9), 16, 4), ((12, 10, 8), 4, 2),
                                             ((33, 17, 8), 132, 6)])
def test_tiles_of_the_host_chooser(shape, n_sm, ctas):
    """sa_tile_choose: a tile that fits the shared buffers, covers the block in at most one wave of resident CTAs where the
    block allows it, and gives the oracle's row"""
    L = C.CDLL(_build())
    out = (C.c_int * 4)()
    assert L.emul_sa_choose(shape[0], shape[1], shape[2], shape[2], n_sm, ctas, out) == 0
    TX, TY, kc, nT = list(out)
    assert nT == TX * TY <= 128 and TX * 8 % 128 == 0 and 1 <= kc <= shape[2]
    tiles = -(-shape[0] // TX) * -(-shape[1] // TY)
    if tiles <= n_sm * ctas:
        assert tiles * -(-shape[2] // kc) <= n_sm * ctas
    if shape[0] * shape[1] * shape[2] > 200000:
        return    # the bench block: the chooser only (the oracle's residual of it takes too long here)
    prm, hb = case(*shape)
    ho = oracle_residual(prm, hb, FLOW | TURB)
    _check(hb, run_emul(prm, hb, 0, 0, 0, n_sm=n_sm, ctas=ctas), ho.dw[..., 5])


def test_emulated_sa_row_in_low_reynolds_regime():
    """low_reynolds (tests/regimes.py): the diffusion of nt is a large share of the row, so a face quantity carried or
    shared wrongly cannot hide in it"""
    import regimes as R
    from test_regimes_reach import assert_reaches

    prm, hb = R.regime_case("low_reynolds", (12, 10, 8))
    assert_reaches(prm, hb, "low_reynolds", ["low_cell_re"])
    ho = oracle_residual(prm, hb, FLOW | TURB)
    for tile in ((7, 4, 3), (16, 8, 1)):
        _check(hb, run_emul(prm, hb, *tile), ho.dw[..., 5])


_ORACLE = {}


def _oracle_row(shape):
    if shape not in _ORACLE:
        prm, hb = case(*shape)
        _ORACLE[shape] = (prm, hb, oracle_residual(prm, hb, FLOW | TURB).dw[..., 5])
    return _ORACLE[shape]


@pytest.mark.parametrize("config", SC.CONFIGS, ids=SC.config_id)
def test_emulated_sa_row_configurations(config):
    """the configuration matrix tests/test_sa_tile_gpu.py runs on the device, with the same plane-by-plane comparison"""
    shape, tile = config
    prm, hb, want = _oracle_row(shape)
    ow = hb.d.owned()
    SC.assert_sa_planes(run_emul(prm, hb, *tile)[ow], want[ow])


@pytest.mark.parametrize("shape,n_sm,ctas", [((96, 72, 64), 132, 3), ((128, 128, 64), 132, 3), ((160, 160, 144), 132, 3),
                                             ((37, 13, 17), 132, 3), ((37, 13, 17), 1, 3), ((33, 9, 23), 5, 3),
                                             ((24, 16, 12), 5, 2), ((129, 17, 16), 132, 3), ((96, 97, 9), 132, 3)])
def test_restated_chooser_is_the_host_chooser(shape, n_sm, ctas):
    """sa_configs.sa_tile_choose (which the device tests use to predict launches) is sa_tile_choose, and the bench picks
    of sa_configs.BENCH_PICKS are what it gives"""
    L = C.CDLL(_build())
    out = (C.c_int * 4)()
    assert L.emul_sa_choose(shape[0], shape[1], shape[2], shape[2], n_sm, ctas, out) == 0
    assert tuple(out)[:3] == SC.sa_tile_choose(shape, shape[2], n_sm, ctas)
    if shape in SC.BENCH_PICKS and (n_sm, ctas) == (SC.H100_SMS, SC.SA_CTAS_PER_SM):
        assert tuple(out)[:3] == SC.BENCH_PICKS[shape]
