"""CPU emulation of the tile kernel (adflow_b200/csrc/fused_kernels.cuh) against the oracle.

The kernel's per-thread phase functions are plain __host__ __device__ code; tests/emul/fused_emul.cu runs them thread
by thread with the shared-memory tiles in host memory.  This checks the tile logic (index maps, halos, k marching,
flux exchange, chunk prologue) for several tile shapes without a GPU; the GPU suite checks the kernel itself."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

from adflow_b200._lib import AdfbParams  # noqa: F401  (ctypes struct)
from util import FLOW, TURB, case, oracle_residual, rel_l2

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "emul", "fused_emul.cu")
SO = os.path.join(HERE, "emul", "libfused_emul%s.so" % os.environ.get("FT_EMUL_FLAGS", "").replace("-D", "_").replace("=", "").replace(" ", ""))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def _build():
    deps = [SRC] + [os.path.join(HERE, "..", "adflow_b200", "csrc", f) for f in ("fused_kernels.cuh", "adfb_common.cuh", "geom_cell.cuh")]
    if os.path.exists(SO) and all(os.path.getmtime(SO) > os.path.getmtime(f) for f in deps):
        return SO
    if not (os.path.exists(NVCC) or shutil.which("nvcc")):
        pytest.skip("nvcc not available")
    subprocess.check_call([NVCC, "-O1", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", "-gencode", "arch=compute_90a,code=sm_90a"]
                          + os.environ.get("FT_EMUL_FLAGS", "").split() + ["-o", SO, SRC])
    return SO


class EmulArrays(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("w", "p", "rlv", "rev", "x", "si", "sj", "sk", "vol", "aa", "ss", "radI", "radJ", "radK", "dw", "fw",
                                          "ssum", "sv", "ovol", "vn", "porI", "porJ", "porK", "iblank")]


def run_emul(prm, hb, ho, TX, TY, kc, rfil=1.0, do_diss=1, merged=1, persist_fw=0, fw=None):
    """flow rows of the residual by the emulated tile kernel; ss/aa/rad are taken from the oracle run `ho`"""
    L = C.CDLL(_build())
    d = hb.d
    N = (d.ib + 1) * (d.jb + 1) * (d.kb + 1)
    keep = {}

    def arr(name, a):
        a = np.asfortranarray(a)
        keep[name] = a
        return a.ctypes.data

    ea = EmulArrays()
    for n in ("w", "p", "rlv", "rev", "x", "si", "sj", "sk", "vol", "porI", "porJ", "porK", "iblank"):
        setattr(ea, n, arr(n, getattr(hb, n)))
    for n in ("aa", "ss", "radI", "radJ", "radK"):
        setattr(ea, n, arr(n, getattr(ho, n)))
    dw = np.zeros(hb.dw.shape, order="F")
    fwa = np.zeros(d.box + (5,), order="F") if fw is None else np.asfortranarray(fw.copy())
    keep["dw"], keep["fw"] = dw, fwa
    ea.dw, ea.fw = dw.ctypes.data, fwa.ctypes.data
    for n, nc in (("ssum", 9), ("sv", 9), ("ovol", 1), ("vn", 12)):
        setattr(ea, n, arr(n, np.zeros(N * nc)))
    L.emul_flowres.argtypes = [C.c_int] * 3 + [C.c_void_p, C.c_void_p] + [C.c_int] * 3 + [C.c_double] + [C.c_int] * 3
    rc = L.emul_flowres(d.nx, d.ny, d.nz, C.byref(prm), C.byref(ea), TX, TY, kc, rfil, do_diss, merged, persist_fw)
    assert rc == 0
    return dw, fwa


@pytest.mark.parametrize("shape,tile", [((12, 10, 8), (9, 5, 4)), ((12, 10, 8), (13, 11, 8)), ((16, 9, 7), (7, 4, 3)), ((10, 6, 9), (5, 7, 9)),
                                         ((14, 8, 6), (21, 9, 2))])
def test_emulated_tile_kernel_matches_oracle_rans(shape, tile):
    prm, hb = case(*shape)
    ho = oracle_residual(prm, hb, FLOW | TURB)
    dw, _ = run_emul(prm, hb, ho, *tile)
    ow = hb.d.owned()
    for l in range(5):
        assert np.isfinite(dw[ow + (l,)]).all()
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-12, l


@pytest.mark.parametrize("shape,n_sm", [((24, 16, 12), 148), ((20, 14, 9), 148), ((33, 17, 8), 16), ((12, 10, 8), 4),
                                        ((24, 16, 12), 132), ((20, 14, 9), 132)])
def test_tiles_of_the_host_chooser(shape, n_sm):
    """ftile_choose (tile shape and k chunk from the cost model, TMA constraint: odd TX) picks small tiles for small blocks and for
    few SMs; whatever it picks must fit the compile-time arrays, cover the block, and give the oracle's residual."""
    prm, hb = case(*shape)
    L = C.CDLL(_build())
    out = (C.c_int * 4)()
    assert L.emul_choose(shape[0], shape[1], shape[2], 1, n_sm, out) == 0
    TX, TY, kc, nT = list(out)
    assert TX % 2 == 1 and TX >= 3 and TY >= 3 and 1 <= kc <= shape[2] and nT % 32 == 0 and nT <= 256
    ho = oracle_residual(prm, hb, FLOW | TURB)
    dw, _ = run_emul(prm, hb, ho, 0, 0, n_sm)          # TX = 0: the chooser's tile on n_sm SMs
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-12, l


def test_emulated_tile_kernel_euler():
    prm, hb = case(12, 8, 10, {"equationType": "Euler"})
    ho = oracle_residual(prm, hb, FLOW)
    dw, _ = run_emul(prm, hb, ho, 7, 5, 5)
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-12, l


@pytest.mark.parametrize("rfil,do_diss", [(0.56, 1), (0.0, 0), (1.0, 1)])
def test_emulated_tile_kernel_smoother_path(rfil, do_diss):
    """block path of the smoothers: central part in dw, dissipative + viscous part blended into the persistent fw
    (residual_block, src/solver/residuals.F90:4-346)"""
    from oracle.pyoracle import Oracle

    prm, hb = case(12, 10, 8)
    ow = hb.d.owned()
    h2 = hb.copy()
    o = Oracle(h2, prm)
    o.time_step(True)
    h2.fw[...] = np.random.default_rng(1).standard_normal(h2.fw.shape) * 1e-3
    fw0 = h2.fw.copy()
    o.residual_block(rfil)
    hs = oracle_residual(prm, hb, FLOW | TURB)   # ss, aa of the same state; radii from the time step
    hs.radI[...], hs.radJ[...], hs.radK[...] = h2.radI, h2.radJ, h2.radK
    dw, fw = run_emul(prm, hb, hs, 9, 5, 4, rfil=rfil, do_diss=do_diss, merged=0, persist_fw=1, fw=fw0)
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], h2.dw[ow + (l,)]) < 1e-12, l
        assert rel_l2(fw[ow + (l,)], h2.fw[ow + (l,)]) < 1e-12, l


# ---------------------------------------------------------------------------------------------------------------------
# flow regimes the smooth state never reaches (tests/regimes.py): a contact discontinuity caps the JST sensor at 0.25
# and cuts the fourth difference off on its faces.  The tile kernel forms i and j faces in shared memory and k faces in
# registers, so each direction is checked, with the jump inside a tile, on a tile seam (the face between the last
# owned cell of one tile and the first of the next: box index 2 + (T-1)) and one cell past it; for k on a chunk seam.
TILE = (9, 5, 4)
SEAMS = {"contact_i": [2 + (TILE[0] - 1) // 2, 2 + TILE[0] - 1, 3 + TILE[0] - 1],
         "contact_j": [2 + (TILE[1] - 1) // 2, 2 + TILE[1] - 1, 3 + TILE[1] - 1],
         "contact_k": [2 + TILE[2] // 2, 2 + TILE[2], 3 + TILE[2]]}


def _regime_rows_close(hb, regime, at, got, want, tol=1e-12):
    import regimes as R

    ow = hb.d.owned()
    far = None if regime == "supersonic" else R.owned_away_from(hb, regime, at)
    for l in range(5):
        a, b = got[ow + (l,)], want[ow + (l,)]
        assert np.isfinite(a).all(), l
        assert rel_l2(a, b) < tol, (l, rel_l2(a, b))
        if far is not None:    # a jump cell's residual can dwarf the rest: hold the cells away from it on their own
            assert rel_l2(a[far], b[far]) < tol, ("away from the jump", l, rel_l2(a[far], b[far]))


REGIME_CASES = [(r, at) for r in ("contact_i", "contact_j", "contact_k") for at in SEAMS[r]] + [("supersonic", None)]


@pytest.mark.parametrize("regime,at", REGIME_CASES)
def test_emulated_tile_kernel_in_regimes(regime, at):
    import regimes as R
    from test_regimes_reach import assert_reaches

    prm, hb = R.regime_case(regime, (12, 10, 8), at=at)
    assert_reaches(prm, hb, regime, ["sensor_cap_" + a for a in ("ijk" if regime == "supersonic" else regime[-1])])
    ho = oracle_residual(prm, hb, FLOW | TURB)
    dw, _ = run_emul(prm, hb, ho, *TILE)
    _regime_rows_close(hb, regime, at, dw, ho.dw)


@pytest.mark.parametrize("regime,at", REGIME_CASES)
def test_emulated_smoother_path_in_regimes(regime, at):
    """merged = 0, persistent fw (the RK / DADI block path) with rFil 0.56: the blend of the capped dissipation"""
    import regimes as R
    from oracle.pyoracle import Oracle

    prm, hb = R.regime_case(regime, (12, 10, 8), at=at)
    h2 = hb.copy()
    o = Oracle(h2, prm)
    o.time_step(True)
    h2.fw[...] = np.random.default_rng(1).standard_normal(h2.fw.shape) * 1e-3
    fw0 = h2.fw.copy()
    o.residual_block(0.56)
    hs = oracle_residual(prm, hb, FLOW | TURB)
    hs.radI[...], hs.radJ[...], hs.radK[...] = h2.radI, h2.radJ, h2.radK
    dw, fw = run_emul(prm, hb, hs, *TILE, rfil=0.56, do_diss=1, merged=0, persist_fw=1, fw=fw0)
    _regime_rows_close(hb, regime, at, dw, h2.dw)
    _regime_rows_close(hb, regime, at, fw, h2.fw)
