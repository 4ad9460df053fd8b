"""The tridiagonal line solves against an exact solve, line by line.

1. The partitioned Thomas solver (adflow_b200/csrc/tridiag_part.cuh, Wang's partition method over P lanes of a warp) on
   its own: tests/kern/part_thomas_harness.cu runs PartThomas<8,12>, <8,16> and <16,16> with the lane mapping of
   k_sa_thomas_part on every line length the SA dispatch sends each of them, on rows built to be hard for a partitioned
   solve, and every line is compared with the exact solution.  The partitioned solve re-associates the elimination, so
   it is held to a multiple of the error the sequential Thomas algorithm (the oracle's tridiagsolve) makes on the same
   line, not to the oracle's bits.
2. The DADI and SA sweeps through the C ABI against the oracle at every length where their dispatch changes kernel,
   compared line by line in each of the three directions (one wrong chunk seam in one line cannot hide under a norm over
   the block), with a kernel trace that shows which solver each length took."""
import contextlib
import ctypes as C
import os
import shutil
import subprocess
from fractions import Fraction

import numpy as np
import pytest

from util import case, rel_l2, rel_max

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "kern", "part_thomas_harness.cu")
CSRC = os.path.join(HERE, "..", "adflow_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")

# PartThomas<P, M> instantiations and the line lengths the SA dispatch (sa_kernels.cuh, launch_sa_block) sends them
INSTANCES = {(8, 12): range(16, 97), (8, 16): range(97, 129), (16, 16): range(129, 257)}
INST_IDS = ["%d_%d" % pm for pm in INSTANCES]

# Bound of the partitioned solve, line by line: max|x - x*| / max|x*| <= max(PART_FACTOR * (the same ratio of the sequential
# Thomas algorithm on that line), PART_FLOOR), x* the exact solution.  Measured on an H100 (80 GB HBM3) over 75 399 lines:
# every dispatched length with the line counts and row families below, and <8,16> at 96, <16,16> at 128 rows (DESIGN.md,
# after the kernel table).  On
# lines where the sequential error is at least 1e-15 the partitioned error was at most 8.3 times it (the random-sign
# dominant rows of <16,16>; at most 3.8 times on the other families), and on lines where it is below 1e-15 the partitioned
# error was at most 1.3e-14 (the same rows; 8.1e-15 on the others).  The constants are those with a margin of 2.
PART_FACTOR = 16.0
PART_FLOOR = 2.5e-14


# ---------------------------------------------------------------------------------------------------------------------
# the harness
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    if not (os.path.exists(NVCC) or shutil.which("nvcc")):
        pytest.skip("nvcc not available")
    so = str(tmp_path_factory.mktemp("part_thomas") / "libpart_thomas_harness.so")
    # the library's own flags (adflow_b200/build.py): the same contraction of the arithmetic into FMAs
    subprocess.check_call([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
                           "-o", so, SRC])
    L = C.CDLL(so)
    L.harness_part_lanes.argtypes = [C.c_int]
    L.harness_part_thomas.argtypes = [C.c_int] * 2 + [C.c_void_p] * 5 + [C.c_int] * 3
    L.harness_part_chunks.argtypes = [C.c_int] * 3 + [C.c_void_p]
    return L


def part_lanes(nl):
    """adfb_part_lanes (adfb_common.cuh), restated"""
    return 8 if 16 <= nl <= 128 else (16 if 128 < nl <= 256 else 0)


def sa_kernel(nl):
    """the line solver launch_sa_block picks for lines of nl cells, restated"""
    part = part_lanes(nl)
    if part == 8:
        return "k_sa_thomas_part<8,12>" if nl <= 96 else "k_sa_thomas_part<8,16>"
    return "k_sa_thomas_part<16,16>" if part == 16 else "k_sa_thomas"


def chunks(n, P):
    """PartThomas<P, M>::chunk, restated: [(start, len)] of the P chunks of an n-row system"""
    return [(p * n // P, (p + 1) * n // P - p * n // P) for p in range(P)]


def part_solve(L, P, M, a, b, c, d):
    """the harness on the systems of the rows of a, b, c, d (nLines x n); the lanes of the surplus of the last warp must not
    store, so a guard of NaN after the last line comes back NaN"""
    nLines, n = b.shape
    guard = 64
    x = np.full(nLines * n + guard, np.nan)
    arr = [np.ascontiguousarray(v, dtype=np.float64) for v in (a, b, c, d)]
    rc = L.harness_part_thomas(P, M, *[v.ctypes.data for v in arr], x.ctypes.data, n, nLines, guard)
    assert rc == 0, "harness_part_thomas<%d,%d>: error %d" % (P, M, rc)
    assert np.isnan(x[nLines * n:]).all(), "a lane stored past the last line"
    return x[:nLines * n].reshape(nLines, n)


# ---------------------------------------------------------------------------------------------------------------------
# the exact reference
def _int_row(vals):
    """the row times the power of two that makes every entry an integer (a row scale leaves the solution unchanged)"""
    fr = [Fraction(float(v)) for v in vals]
    den = max(f.denominator for f in fr)
    return [int(f * den) for f in fr]


def exact_fraction(a, b, c, d):
    """Thomas elimination in rational arithmetic on the double rows, the solution rounded once to double (slow: small
    systems)"""
    n = len(b)
    A, B, Cc, D = ([Fraction(float(v)) for v in r] for r in (a, b, c, d))
    cp, dp = [Fraction(0)] * n, [Fraction(0)] * n
    for i in range(n):
        piv = B[i] - (A[i] * cp[i - 1] if i else 0)
        cp[i] = Cc[i] / piv
        dp[i] = (D[i] - (A[i] * dp[i - 1] if i else 0)) / piv
    x = [Fraction(0)] * n
    x[-1] = dp[-1]
    for i in range(n - 2, -1, -1):
        x[i] = dp[i] - cp[i] * x[i + 1]
    return np.array([float(v) for v in x])


_BITS = 320


def _near(num, den):
    """the rational num / den (integers) truncated to _BITS significant bits"""
    if den < 0:
        num, den = -num, -den
    if num == 0:
        return Fraction(0)
    sh = _BITS - (abs(num).bit_length() - den.bit_length())
    return Fraction((num << sh) // den, 1 << sh) if sh >= 0 else Fraction((num // (den << -sh)) << -sh)


def exact_solve(a, b, c, d):
    """x* of one system, rounded once to double.  The elimination is exact: with every row scaled to integers, the pivots
    are P_i / P_(i-1) and the eliminated right-hand sides g_i / P_i of the integer continuants
        P_i = b_i P_(i-1) - a_i c_(i-1) P_(i-2),   g_i = d_i P_(i-1) - a_i g_(i-1).
    The back substitution x_i = g_i / P_i - (c_i P_(i-1) / P_i) x_(i+1) carries 320-bit significands, and |c_i P_(i-1) /
    P_i| <= 1 on a diagonally dominant system, so x* is within n 2**-318 max|x| of the exact solution before its rounding:
    the same doubles as exact_fraction (checked), at a cost linear in n."""
    n = len(b)
    A, B, Cc, D = zip(*[_int_row((a[i], b[i], c[i], d[i])) for i in range(n)])
    P, g = [0] * n, [0] * n
    pm2, pm1 = 0, 1
    for i in range(n):
        P[i] = B[i] * pm1 - (A[i] * Cc[i - 1] * pm2 if i else 0)
        g[i] = D[i] * pm1 - (A[i] * g[i - 1] if i else 0)
        pm2, pm1 = pm1, P[i]
    assert all(P), "singular leading block"
    x = [0.0] * n
    xn = _near(g[-1], P[-1])
    x[-1] = float(xn)
    for i in range(n - 2, -1, -1):
        v = _near(g[i], P[i]) - _near(Cc[i] * (P[i - 1] if i else 1), P[i]) * xn
        xn = _near(v.numerator, v.denominator)
        x[i] = float(xn)
    return np.array(x)


def thomas_seq(a, b, c, d):
    """tridiagsolve (residuals.F90:1750-1783, oracle/adflow_oracle_smooth.c) restated on rows 0..n-1 of each line: forward
    elimination with the reciprocal of the pivot, back substitution"""
    a, b, c, d = (np.asarray(v, dtype=np.float64) for v in (a, b, c, d))
    dd, ff = c.copy(), d.copy()
    n = b.shape[-1]
    d0 = 1.0 / b[..., 0]
    dd[..., 0] *= d0
    ff[..., 0] *= d0
    for m in range(1, n):
        d0 = 1.0 / (b[..., m] - a[..., m] * dd[..., m - 1])
        ff[..., m] = (ff[..., m] - a[..., m] * ff[..., m - 1]) * d0
        dd[..., m] *= d0
    for m in range(n - 2, -1, -1):
        ff[..., m] = ff[..., m] - dd[..., m] * ff[..., m + 1]
    return ff


def line_err(x, xs):
    """max|x - x*| / max|x*| of each line"""
    return np.abs(x - xs).max(axis=-1) / np.abs(xs).max(axis=-1)


# ---------------------------------------------------------------------------------------------------------------------
# row families
def _dominant(rng, n, lo, hi):
    """random signs and sizes, b = (|a| + |c|)(1 + r) with the relative margin r log-uniform in [10**lo, 10**hi]"""
    a = rng.uniform(-1, 1, n) * 10.0 ** rng.uniform(-1, 1, n)
    c = rng.uniform(-1, 1, n) * 10.0 ** rng.uniform(-1, 1, n)
    a[0] = c[-1] = 0.0
    b = (np.abs(a) + np.abs(c)) * (1.0 + 10.0 ** rng.uniform(lo, hi, n))
    return a, b, c, rng.uniform(-1, 1, n)


def _sa_rows(rng, n, up=True):
    """the sign structure of the SA DD-ADI rows (a, c <= 0, b >= |a| + |c|) with off-diagonals that change by 1e10 along the
    line, as the diffusion coefficients do across the 1e-5 first cell of synthetic.node_coordinates"""
    s = 10.0 ** (10.0 * np.arange(n) / (n - 1))
    s = s if up else s[::-1]
    a = -s * rng.uniform(0.5, 1.5, n)
    c = -s * rng.uniform(0.5, 1.5, n)
    a[0] = c[-1] = 0.0
    b = (np.abs(a) + np.abs(c)) * (1.0 + 10.0 ** rng.uniform(-8, 0, n)) + 1.0
    return a, b, c, rng.uniform(-1, 1, n) * s


def families(n, P, seed):
    """[(family, a, b, c, d)]: dominant rows over the whole margin range, at the tightest and at the loosest margin; SA
    rows stretched up and down the line; zero off-diagonals on the seams of chunks P/2-1 | P/2 and 1 | 2 and inside chunks
    2 and 3; a right-hand side in one chunk only (the middle one, the last one)"""
    rng = np.random.default_rng(seed)
    ch = chunks(n, P)
    out = [("dominant", *_dominant(rng, n, -10, 6)), ("sa_stretched", *_sa_rows(rng, n, True)),
           ("dominant", *_dominant(rng, n, -10, -10))]
    a, b, c, d = _dominant(rng, n, -3, 1)
    s0, m0 = ch[P // 2]
    a[s0] = c[s0 - 1] = 0.0                    # the seam P/2-1 | P/2 cut both ways
    c[ch[1][0] + ch[1][1] - 1] = 0.0           # 1 | 2 one way only
    out.append(("zero_offdiag_seam", a, b, c, d))
    a, b, c, d = _sa_rows(rng, n, False)
    s2, m2 = ch[2]
    s3, m3 = ch[3]
    a[s2 + m2 // 2] = 0.0
    c[s3 + m3 // 2] = 0.0
    a[s3 + 1] = c[s3 + 1] = 0.0
    out.append(("zero_offdiag_inside", a, b, c, d))
    for q in (P // 2, P - 1):
        a, b, c, d = _sa_rows(rng, n, q == P - 1)
        s, m = ch[q]
        keep = np.zeros(n, bool)
        keep[s:s + m] = True
        out.append(("rhs_in_one_chunk", a, b, c, np.where(keep, d, 0.0)))
    out.append(("dominant", *_dominant(rng, n, 6, 6)))
    out.append(("sa_stretched", *_sa_rows(rng, n, False)))
    return out


def pool(n, P, seed):
    """the systems of a length: (family names, a, b, c, d stacked), their exact solutions and the sequential errors"""
    fam = families(n, P, seed)
    names = [f[0] for f in fam]
    a, b, c, d = (np.array([f[q] for f in fam]) for q in range(1, 5))
    xs = np.array([exact_solve(*r) for r in zip(a, b, c, d)])
    return names, (a, b, c, d), xs, line_err(thomas_seq(a, b, c, d), xs)


def bound(seq_err):
    return np.maximum(PART_FACTOR * seq_err, PART_FLOOR)


# ---------------------------------------------------------------------------------------------------------------------
# host only
def test_dispatch_and_chunks(harness):
    """the restated dispatch is the library's adfb_part_lanes, every partitioned length is dispatched to the instantiation
    this file tests it on, and every chunk of every such length has 2 <= m <= M rows (PartThomas::solve's precondition)"""
    for n in range(1, 1025):
        assert harness.harness_part_lanes(n) == part_lanes(n), n
        k = sa_kernel(n)
        pm = [pm for pm, r in INSTANCES.items() if n in r]
        assert (k == "k_sa_thomas") == (not pm), n
        if not pm:
            continue
        (P, M), = pm
        assert k == "k_sa_thomas_part<%d,%d>" % (P, M) and part_lanes(n) == P, n
        ch = chunks(n, P)
        assert ch[0][0] == 0 and sum(m for _, m in ch) == n and all(ch[q][0] + ch[q][1] == ch[q + 1][0] for q in range(P - 1))
        assert all(2 <= m <= M for _, m in ch), (n, P, M, ch)


def test_exact_reference():
    """exact_solve gives the doubles of rational Thomas elimination and agrees with numpy.linalg.solve; the sequential
    double Thomas comes within 1e-14 of it on the M-matrix rows of the SA families"""
    for n, P in ((16, 8), (37, 8), (64, 8), (40, 16)):
        for q, (name, a, b, c, d) in enumerate(families(n, P, n)):
            xs = exact_solve(a, b, c, d)
            assert np.array_equal(xs, exact_fraction(a, b, c, d)), (n, name)
            Mx = np.diag(b) + np.diag(a[1:], -1) + np.diag(c[:-1], 1)
            cond = np.linalg.cond(Mx, np.inf)
            assert np.abs(np.linalg.solve(Mx, d) - xs).max() <= 10 * cond * 2.0 ** -52 * np.abs(xs).max(), (n, name)
            seq = line_err(thomas_seq(a, b, c, d), xs)
            if name in ("sa_stretched", "rhs_in_one_chunk"):
                assert 0 <= seq < 1e-14, (n, name, seq)


def test_exact_reference_catches_a_perturbed_row():
    """a change of one ulp in one row moves x* (the reference resolves what the bound asks of the kernel)"""
    name, a, b, c, d = families(64, 8, 3)[1]
    xs = exact_solve(a, b, c, d)
    d2 = d.copy()
    d2[40] = np.nextafter(d2[40], np.inf)
    assert not np.array_equal(exact_solve(a, b, c, d2), xs)


# ---------------------------------------------------------------------------------------------------------------------
# the partitioned solve on the GPU
def _check_part(L, P, M, n, pl, nLines, off, want_lines=None):
    names, (a, b, c, d), xs, seq = pl
    sel = (np.arange(nLines) + off) % len(names)
    x = part_solve(L, P, M, a[sel], b[sel], c[sel], d[sel])
    assert np.isfinite(x).all(), (P, M, n, nLines)
    err = line_err(x, xs[sel])
    bad = np.nonzero(err > bound(seq[sel]))[0]
    if bad.size:
        q = bad[np.argmax(err[bad] / bound(seq[sel][bad]))]
        cell = int(np.argmax(np.abs(x[q] - xs[sel[q]])))
        chunk = next(p for p, (s, m) in enumerate(chunks(n, P)) if s <= cell < s + m)
        pytest.fail("PartThomas<%d,%d> n=%d, %d lines: line %d (%s) error %.3e > bound %.3e (sequential %.3e); worst row %d, chunk %d"
                    % (P, M, n, nLines, q, names[sel[q]], err[q], bound(seq[sel[q]]), seq[sel[q]], cell, chunk))
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("pm", list(INSTANCES), ids=INST_IDS)
def test_partitioned_thomas_every_length(cuda_lib, harness, pm):
    """every length of the instantiation's dispatch range, 1, LS-1, LS, LS+1 and 301 lines (a partial last warp and lanes
    that redo the last line), each line against its exact solution"""
    P, M = pm
    LS = 32 // P
    for n in INSTANCES[pm]:
        pl = pool(n, P, 1000 * P + n)
        for q, nLines in enumerate(sorted({1, max(LS - 1, 1), LS, LS + 1, 301})):
            _check_part(harness, P, M, n, pl, nLines, off=q + n)


@pytest.mark.gpu
def test_partitioned_thomas_device_chunks(cuda_lib, harness):
    """PartThomas::chunk on the device is the restatement the host tests check"""
    for (P, M), r in INSTANCES.items():
        for n in (r[0], r[-1], (r[0] + r[-1]) // 2):
            out = (C.c_int * (2 * P))()
            assert harness.harness_part_chunks(P, M, n, out) == 0
            assert [(out[2 * p], out[2 * p + 1]) for p in range(P)] == chunks(n, P), (P, M, n)


@pytest.mark.gpu
@pytest.mark.parametrize("n,pms", [(96, ((8, 12), (8, 16))), (128, ((8, 16), (16, 16)))])
def test_partitioned_thomas_instantiations_agree(cuda_lib, harness, n, pms):
    """<8,16> at 96 rows and <16,16> at 128 (outside their dispatch ranges, inside their capacity) meet the bound against the
    exact solution, and agree with the instantiation the length is dispatched to to the same bound"""
    pl = pool(n, pms[0][0], 7 * n)
    names, _, xs, seq = pl
    nLines = 3 * len(names)
    sel = np.arange(nLines) % len(names)
    xa, xb = (_check_part(harness, P, M, n, pl, nLines, 0) for P, M in pms)
    dev = np.abs(xa - xb).max(axis=-1) / np.abs(xs[sel]).max(axis=-1)
    assert (dev <= bound(seq[sel])).all(), (n, pms, dev.max())
    if pms[1][0] != pms[0][0]:   # and on rows whose seams and zeros follow its own 16 chunks
        _check_part(harness, *pms[1], n, pool(n, pms[1][0], 7 * n), nLines, 0)


# ---------------------------------------------------------------------------------------------------------------------
# the sweeps of the library, line by line
@contextlib.contextmanager
def traced(s, seen):
    """collect into `seen` the canonical names (kernel_table.canonical) of the kernels launched inside the block; the
    context's CUDA graphs are bypassed meanwhile (per-kernel timing on), so that every launch is traced by itself"""
    import torch
    from torch.profiler import ProfilerActivity, profile

    from kernel_table import canonical

    s.L.adfb_set_timing(1)
    try:
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            yield
            s.synchronize()
            torch.cuda.synchronize()
    finally:
        s.L.adfb_set_timing(0)
    seen.update(canonical(e.name) for e in prof.events())
    seen.discard(None)


def assert_lines_close(got, want, tol, what):
    """every line of each direction: |got - want| <= tol max over the line of |want|; got, want over the owned cells"""
    assert np.isfinite(got).all(), what
    for ax, dname in enumerate("ijk"):
        g, w = np.moveaxis(got, ax, -1), np.moveaxis(want, ax, -1)
        scale = np.abs(w).max(axis=-1, keepdims=True)
        excess = np.abs(g - w) - tol * scale
        if (excess > 0).any():
            rel = np.abs(g - w) / np.where(scale > 0, scale, 1.0)
            line = np.unravel_index(np.argmax(np.where(excess > 0, rel, -1.0)), rel.shape)
            cell = list(line[:-1])
            cell.insert(ax, line[-1])
            other = "".join(n for n in "ijk" if n != dname)
            pytest.fail("%s: %s line at %s = %s (%d cells): worst cell (i,j,k) = %s, |got - want| = %.3e = %.3e of the line's max "
                        "%.3e (tol %.0e)" % (what, dname, other, tuple(int(v) + 2 for v in line[:-1]), got.shape[ax],
                                             tuple(int(v) + 2 for v in cell), abs(g[line] - w[line]), rel[line], scale[line[:-1]][0], tol))


SA_SOLVERS = {"k_sa_thomas", "k_sa_thomas_part<8,12>", "k_sa_thomas_part<8,16>", "k_sa_thomas_part<16,16>"}


def _sa_line_by_line(prm, hb0):
    """_sa_solve_matches of test_regimes_gpu.py (one turbSolveDDADI sub-iteration against the oracle's sa_block), with the
    change of nuTilde held line by line; returns the SA line solvers the device launched"""
    from adflow_b200.solver import ADFLOW_B200
    from oracle.pyoracle import Oracle

    ho = hb0.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.sa_block()
    seen = set()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb0)
        s.applyBCs(True, True)
        with traced(s, seen):
            s.turbSolveDDADI(1)
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb0.d.owned()
    assert rel_l2(dw[ow + (5,)], ho.dw[ow + (5,)]) < 1e-10
    dn, do = w[ow + (5,)] - hb0.w[ow + (5,)], ho.w[ow + (5,)] - hb0.w[ow + (5,)]
    assert np.abs(do).max() > 0
    assert rel_l2(dn, do) < 1e-9, rel_l2(dn, do)
    assert_lines_close(dn, do, 1e-9, "SA state change")
    assert rel_max(w[..., 5], ho.w[..., 5]) < 1e-10
    d = hb0.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    assert rel_max(rev[c1], ho.rev[c1]) < 1e-10
    return seen & SA_SOLVERS


# The long direction takes each length on both sides of every boundary of the SA dispatch (15 | 16, 96 | 97, 128 | 129,
# 256 | 257); the cross-section is 5 x 7 = 35 lines, not a multiple of the 4 or 2 lines a warp of the partitioned solvers
# takes, so the last warp has lanes that redo the last line.
SA_LENGTHS = (15, 16, 17, 95, 96, 97, 128, 129, 255, 256, 257)


@pytest.mark.gpu
@pytest.mark.parametrize("axis", [0, 1, 2], ids=["i", "j", "k"])
@pytest.mark.parametrize("nl", SA_LENGTHS)
def test_sa_ddadi_line_by_line(cuda_lib, nl, axis):
    shape = [5, 7]
    shape.insert(axis, nl)
    prm, hb = case(*shape)
    assert _sa_line_by_line(prm, hb) == {sa_kernel(n) for n in shape}, (shape, nl)


# The O-grid of tests/meshes.py (stiff wall-normal lines of 1e4 aspect ratio along k) and its axis permutations, the stiff
# lines along i and j, with radial line lengths at the ends of each partitioned range; 5 x 7 lines.
OGRID_RADIAL = (16, 96, 97, 128, 129, 256)


@pytest.mark.gpu
@pytest.mark.parametrize("radial", OGRID_RADIAL)
@pytest.mark.parametrize("name", ["o_grid", "o_grid_jk", "o_grid_ki"])
def test_sa_ddadi_line_by_line_o_grid(cuda_lib, name, radial):
    from test_mesh_topologies_gpu import block

    prm, hb, _ = block(name, shape=(5, 7, radial))
    shape = (hb.d.nx, hb.d.ny, hb.d.nz)
    assert radial in shape
    assert _sa_line_by_line(prm, hb) == {sa_kernel(n) for n in shape}, (name, shape)


def _dadi_line_by_line(prm, hb):
    """test_dadi_line_counts_and_lengths of test_regimes_gpu.py (one DADI step against the oracle's), with the change of each
    variable held line by line; returns the DADI line solvers the device launched"""
    from adflow_b200.solver import ADFLOW_B200
    from test_regimes_gpu import _smoother_start

    ho, o = _smoother_start(prm, hb)
    o.dadi_step()
    seen = set()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        with traced(s, seen):
            s.dadiStep()
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        dv, do = w[ow + (l,)] - hb.w[ow + (l,)], ho.w[ow + (l,)] - hb.w[ow + (l,)]
        assert rel_l2(dv, do) < 1e-9, ("state change", l, rel_l2(dv, do))
        assert_lines_close(dv, do, 1e-9, "DADI state change of variable %d" % l)
    assert rel_max(p, ho.p) < 1e-11
    return seen & {"k_dadi_thomas", "k_dadi_thomas_tile"}


# k_dadi_thomas_tile walks the i lines 32 to a warp in chunks of ADFB_DT_CH = 8 cells: 31, 32, 33 and 65 lines (a partial
# warp, one full warp, one line over, two warps and one line) of 7, 8, 9, 16 and 17 cells (a short chunk, whole chunks, one
# cell over).  The j and k lines take k_dadi_thomas.
@pytest.mark.gpu
@pytest.mark.parametrize("n1", (31, 32, 33, 65))
@pytest.mark.parametrize("nl", (7, 8, 9, 16, 17))
def test_dadi_line_by_line(cuda_lib, nl, n1):
    prm, hb = case(nl, n1, 5)
    assert _dadi_line_by_line(prm, hb) == {"k_dadi_thomas", "k_dadi_thomas_tile"}


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["o_grid", "o_grid_jk", "o_grid_ki"])
def test_dadi_line_by_line_o_grid(cuda_lib, name):
    """the stiff radial lines (17 cells: two chunks and one cell) along k, i and j; 33 circumferential lines"""
    from test_mesh_topologies_gpu import block

    prm, hb, _ = block(name, shape=(5, 33, 17))
    assert _dadi_line_by_line(prm, hb) == {"k_dadi_thomas", "k_dadi_thomas_tile"}
