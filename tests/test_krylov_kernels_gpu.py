"""The vector kernels of the device GMRES (adflow_b200/csrc/krylov_kernels.cuh) on their own, against exactly rounded
results: tests/kern/krylov_harness.cu launches them as adfb_gmres_solve does.

k_multidot + k_multidot_final form V_i . w by per-thread serial sums over a grid-stride loop (ADFB_GMRES_PARTS CTAs of
256 threads), a 256-way tree in each CTA and a 256-way tree over the CTAs' partials.  Every term therefore passes through
at most L + 17 roundings, L = ceil(n / 65536) the length of a thread's serial sum (its product, the serial sum, two trees
of depth 8), and the dot is held to the forward bound of that order: |dot - exact| <= gamma_(L+17) sum |V_i[q] w[q]|,
gamma_d = d u / (1 - d u), u = 2^-53.  The exact dots are math.fsum of the products, which are exact doubles because
every entry of w is a power of two and every product stays inside the normal range.  The order must not depend on nv or
on the call, so each dot is also compared bit for bit across nv and across repeated calls.  k_axpy_many is held to the
bound of its own order (one fused multiply-add per vector) against extended precision, k_scale_to to numpy's bits."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "kern", "krylov_harness.cu")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
PARTS, THREADS = 256, 256           # ADFB_GMRES_PARTS and the CTA size of k_multidot
U = 2.0 ** -53

SIZES = [1, 255, 256, 257, 65535, 65536, 65537, 3 * 65536 + 17]
NV = [1, 2, 127, 128]
HUGE = 30_000_017                   # ~3e7: a serial sum of 458 terms per thread


@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not (os.path.exists(NVCC) or shutil.which("nvcc")):
        pytest.skip("nvcc not available")
    so = str(tmp_path_factory.mktemp("krylov") / "libkrylov_harness.so")
    # the library's own flags (adflow_b200/build.py): the same contraction of the arithmetic into FMAs
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-o", so, SRC])
    L = C.CDLL(so)
    L.harness_dots.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]
    L.harness_axpy_many.argtypes = [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_double, C.c_void_p, C.c_longlong, C.c_int]
    L.harness_scale_to.argtypes = [C.c_void_p, C.c_double, C.c_void_p, C.c_longlong, C.c_int]
    return L


def shared_w(rng, n):
    """the w all V_i are dotted with: +-2^e, e in -20..20, so every product V_i[q] w[q] is an exact double"""
    return rng.choice([-1.0, 1.0], n) * np.ldexp(1.0, rng.integers(-20, 21, n))


def operand(rng, n, w, family):
    """one V_i against w: 'normal' standard normal; 'positive' every product > 0 (no cancellation); 'wide' magnitudes
    from 1e-150 to 1e150 with three quarters of the products in pairs p, -p at unrelated places, so the exact dot is the
    few unpaired terms and the rest cancels"""
    if family == "normal":
        return rng.standard_normal(n)
    if family == "positive":
        return np.sign(w) * rng.uniform(0.5, 2.0, n)
    v = rng.choice([-1.0, 1.0], n) * rng.uniform(1, 10, n) * 10.0 ** rng.uniform(-150, 150, n)
    h = 3 * n // 8
    perm = rng.permutation(n)
    a, b = perm[:h], perm[h:2 * h]
    v[b] = -v[a] * w[a] / w[b]          # exact: w is a power of two
    return v


FAMILIES = ["normal", "wide", "positive"]


def exact_dot(v, w):
    return math.fsum((v * w).tolist())


def bound(n, v, w):
    d = -(-n // (PARTS * THREADS)) + 17
    return d * U / (1 - d * U) * float(np.abs(v * w).sum())


def dots(L, V, ld, nv, w, n):
    out = np.full(nv, np.nan)
    rc = L.harness_dots(V.ctypes.data, ld, nv, w.ctypes.data, n, out.ctypes.data)
    assert rc == 0, "harness_dots: error %d" % rc
    return out


def basis(rng, n, nv, ld):
    """nv vectors of n entries at stride ld, the entries past n poisoned with NaN (a read past n shows), the families
    cycling over the vectors; returns V, w, the exact dots and their bounds"""
    w = shared_w(rng, n)
    V = np.full((nv, ld), np.nan)
    for i in range(nv):
        V[i, :n] = operand(rng, n, w, FAMILIES[i % 3])
    return V, w, np.array([exact_dot(V[i, :n], w) for i in range(nv)]), np.array([bound(n, V[i, :n], w) for i in range(nv)])


@pytest.mark.parametrize("n", SIZES)
def test_multidot_against_exact_dots(cuda_lib, harness, n):
    rng = np.random.default_rng(n)
    ld = n + 3                          # ld != n
    V, w, ex, bd = basis(rng, n, max(NV), ld)
    full = dots(harness, V, ld, max(NV), w, n)
    err = np.abs(full - ex)
    assert np.all(err <= bd), (int(np.argmax(err / bd)), (err / bd).max())
    assert np.all(np.isfinite(full))
    # the dot of V_i does not depend on how many vectors share the pass, nor on the call
    for nv in NV:
        assert np.array_equal(dots(harness, V, ld, nv, w, n), full[:nv]), nv
    assert np.array_equal(dots(harness, V, ld, max(NV), w, n), full)
    assert np.array_equal(dots(harness, np.ascontiguousarray(V[4:5]), ld, 1, w, n), full[4:5])


def test_multidot_huge(cuda_lib, harness):
    """n ~ 3e7: 458 terms in each thread's serial sum before the trees; nv = 1 and 2"""
    n = HUGE
    V, w, ex, bd = basis(np.random.default_rng(3), n, 2, n + 1)
    out = dots(harness, V, n + 1, 2, w, n)
    assert np.all(np.abs(out - ex) <= bd), (out, ex, bd)
    assert np.array_equal(dots(harness, V, n + 1, 1, w, n), out[:1])


@pytest.mark.parametrize("n", [257, 65537])
def test_multidot_nan_stays_in_its_dot(cuda_lib, harness, n):
    nv, ld = 127, n + 5
    V, w, _, _ = basis(np.random.default_rng(9), n, nv, ld)
    clean = dots(harness, V, ld, nv, w, n)
    assert np.isfinite(clean).all()
    for i, q in ((0, 0), (63, n // 2), (126, n - 1)):
        Vn = V.copy()
        Vn[i, q] = np.nan
        out = dots(harness, Vn, ld, nv, w, n)
        others = np.arange(nv) != i
        assert np.isnan(out[i]) and np.array_equal(out[others], clean[others]), i
    wn = w.copy()
    wn[n // 3] = np.inf
    Vz = V[:3].copy()
    Vz[:, n // 3] = [1.0, 0.0, -1.0]    # 0 * inf: NaN in that dot only; the others see +-inf
    out = dots(harness, Vz, ld, 3, wn, n)
    assert out[0] == np.inf and np.isnan(out[1]) and out[2] == -np.inf


def _exact_axpy(V, coef, beta, y):
    """beta y + sum_i coef_i V_i, every entry in extended precision and rounded once"""
    LD = np.longdouble
    a = LD(beta) * y.astype(LD) if beta != 0 else np.zeros(y.size, LD)
    for c, v in zip(coef, V):
        a += LD(c) * v.astype(LD)
    return a.astype(np.float64), (abs(beta) * np.abs(y) if beta != 0 else 0) + np.abs(np.asarray(coef)) @ np.abs(V)


@pytest.mark.parametrize("n", [1, 255, 256, 257, 65537])
@pytest.mark.parametrize("nv", [0, 1, 2, 127, 128])
def test_axpy_many(cuda_lib, harness, n, nv):
    rng = np.random.default_rng(n * 7 + nv)
    ld, guard = n + 2, 4
    V = np.full((max(nv, 1), ld), np.nan)
    V[:, :n] = rng.standard_normal((max(nv, 1), n)) * 10.0 ** rng.uniform(-3, 3, (max(nv, 1), 1))
    coef = rng.standard_normal(nv)
    for beta in (0.0, 1.0, -1.0, 0.37):
        y0 = rng.standard_normal(n)
        y = np.concatenate([y0, np.full(guard, 7.5)])
        if beta == 0.0:
            y[:n] = np.nan              # beta = 0 overwrites: the old y must not leak in as 0 * NaN
        rc = harness.harness_axpy_many(V.ctypes.data, ld, nv, coef.ctypes.data, beta, y.ctypes.data, n, guard)
        assert rc == 0, rc
        want, mag = _exact_axpy(V[:nv, :n], coef, beta, y0)
        d = nv + 2
        assert np.all(np.abs(y[:n] - want) <= d * U / (1 - d * U) * mag + 1e-300), (beta, np.max(np.abs(y[:n] - want)))
        assert np.all(y[n:] == 7.5)


@pytest.mark.parametrize("n", [1, 255, 257, 65537, 3 * 65536 + 17])
def test_scale_to(cuda_lib, harness, n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n) * 10.0 ** rng.uniform(-150, 150, n)
    for a in (1.0 / 3.0, -2.5e-7):
        y = np.concatenate([np.full(n, np.nan), np.full(3, 7.5)])
        assert harness.harness_scale_to(x.ctypes.data, a, y.ctypes.data, n, 3) == 0
        assert np.array_equal(y[:n], a * x)       # one rounding per entry: the same bits as numpy
        assert np.all(y[n:] == 7.5)
