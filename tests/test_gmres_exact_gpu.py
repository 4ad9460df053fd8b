"""The device GMRES (adfb_gmres_solve) against the exact GMRES(m) iterates of tests/gmres_ref.py.

The operator is op 2, the block-diagonal time-step matrix T whose blocks the oracle provides, right-preconditioned by a
callback that applies M^-1 block by block on the device vectors (torch).  The callback sets the spectrum of T M^-1:
M^-1 = T^-1 S with S normal and chosen, so that T M^-1 = S up to the rounding of M^-1.  The exact iterates take T and
M^-1 as the doubles they are.

Each x_k is reached as the result of a solve with maxIts = k and rtol = atol = 0, for every k of at least two restart
cycles.  A device iterate is held to the exact one by
  ||x - x_k|| <= X_TOL ||x_k||   and   |resNorm - ||b - A y_k||| <= RES_TOL ||b||,
and everywhere a reported resNorm must not lie below the true residual ||b - T x|| by more than RES_TOL ||b||, and must
be NaN whenever the recurrence or ||b|| is not finite.  The tolerances are measured values with a margin of 2
(DESIGN.md, after the kernel table)."""
import ctypes as C

import numpy as np
import pytest

from adflow_b200._lib import check
from adflow_b200.params import make_ank_params
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
from oracle.pyoracle import Oracle

from gmres_ref import LD, ExactGmres, block_operator
from test_ank_gpu import oracle_blocks
from util import case

pytestmark = pytest.mark.gpu

# Largest deviations from the exact iterates over these tests, measured on an H100 80GB HBM3 at 700 W, times 2
# (DESIGN.md, after the kernel table).  x, per system: 8.8e-15 on the 9 x 8 x 7 block (four distinct eigenvalues; 7.2e-15
# over every iterate at restart 60), 6.6e-16 on one cell, 9.6e-16 on three blocks, 1.2e-10 on the coupled 40 x 32 x 16
# block, whose time-step blocks have condition numbers up to 2e8, so that T (M^-1 v) in double already moves T M^-1 v
# by that much.  resNorm: 1.2e-13 of ||b|| (the four-eigenvalue termination, where the exact residual is 6e-14; at most
# 1.9e-14 elsewhere); a reported residual was never more than 8.1e-15 ||b|| below the true one.
X_TOL = {"single": 1.8e-14, "cell": 1.4e-15, "three": 2.0e-15, "large": 2.4e-10}
RES_TOL = 2.4e-13

SINGLE_ANK = make_ank_params(cfl=3.0, coupled=False, char_time_step="VLR", cflLimit=20.0)
PCFN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong)


# ---------------------------------------------------------------------------------------------------------------------
# operators
def time_step_blocks(prm, ank, hb):
    """BCs, time step and speed of sound of the state in hb (in place, so the device gets the same state); T's blocks"""
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    o.call("orc_speed_of_sound", C.byref(prm))
    return oracle_blocks(prm, ank, hb)


def disc_spectrum(rng, nc, ns, radius):
    """nc normal (ns x ns) blocks Q D Q^T: D holds 2 x 2 rotation-scalings of eigenvalues 1 + r e^(+-i t) filling the
    disc of `radius` about 1 (and one real eigenvalue for odd ns), Q random orthogonal"""
    D = np.zeros((nc, ns, ns))
    for p in range(0, ns - 1, 2):
        r = radius * np.sqrt(rng.uniform(size=nc))
        t = rng.uniform(0.0, np.pi, nc)
        D[:, p, p] = D[:, p + 1, p + 1] = 1.0 + r * np.cos(t)
        D[:, p, p + 1], D[:, p + 1, p] = r * np.sin(t), -r * np.sin(t)
    if ns % 2:
        D[:, -1, -1] = 1.0 + radius * rng.uniform(-1.0, 1.0, nc)
    return _rotate(rng, D)


def few_values_spectrum(rng, nc, ns, values):
    """nc symmetric blocks Q diag(v) Q^T, every eigenvalue one of `values`"""
    D = np.zeros((nc, ns, ns))
    idx = np.arange(ns)
    D[:, idx, idx] = rng.choice(values, (nc, ns))
    D[0, idx[:len(values)], idx[:len(values)]] = values           # every value present
    return _rotate(rng, D)


def _rotate(rng, D):
    Q, _ = np.linalg.qr(rng.standard_normal(D.shape))
    return Q @ D @ np.transpose(Q, (0, 2, 1))


def preconditioner_for(T, S):
    """M^-1 = T^-1 S, block by block: T M^-1 = S to the rounding of M^-1"""
    return np.linalg.solve(T, S)


class DevVec:   # a device pointer as a CUDA array for torch (torch rejects read-only views)
    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 2}


class Precond:
    """out = M^-1 in, block by block, on the device vectors; counts its calls and returns a NaN in one entry on call
    `nan_at`"""

    def __init__(self, Minv, nan_at=None):
        import torch

        self.M = torch.from_numpy(np.ascontiguousarray(Minv)).cuda()
        self.ns = Minv.shape[1]
        self.calls, self.nan_at = 0, nan_at
        self.fn = PCFN(self._apply)

    def _apply(self, ctx, in_ptr, out_ptr, n):
        import torch

        self.calls += 1
        v = torch.as_tensor(DevVec(in_ptr, n), device="cuda").reshape(-1, self.ns)
        out = torch.as_tensor(DevVec(out_ptr, n), device="cuda").reshape(-1, self.ns)
        out.copy_(torch.einsum("qlm,qm->ql", self.M, v))
        if self.calls == self.nan_at:
            out[out.shape[0] // 2, 1] = float("nan")
        torch.cuda.synchronize()
        return 0


# ---------------------------------------------------------------------------------------------------------------------
# device contexts: one live at a time (the library has one per process); tests that share one sit together
_live = {}


@pytest.fixture(scope="module", autouse=True)
def _close_last():
    yield
    _drop()


def _drop():
    for sysm in _live.values():
        sysm.s.close()
    _live.clear()


class System:
    """a context whose time-step matrix is ready, with T's blocks from the oracle"""

    def __init__(self, key, prm, ank, hbs):
        self.key = key
        self.T = np.concatenate([time_step_blocks(prm, ank, hb) for hb in hbs])
        self.ns = self.T.shape[1]
        self.nc = self.T.shape[0]
        self.n = self.nc * self.ns
        self.s = ADFLOW_B200(prm)
        try:
            for hb in hbs:
                self.s.addBlock(hb)
            self.s.ankSetParams(ank)
            self.s.residual(RES_FLOW | RES_TURB | 4)
            self.s.ankTimeStepMat()
        except Exception:
            self.s.close()
            raise

    def solve(self, b, restart, max_its, rtol=0.0, atol=0.0, pc=None):
        b = np.ascontiguousarray(b, dtype=np.float64)
        x = np.zeros_like(b)
        its, rn = C.c_int(-1), C.c_double(-1.0)
        rc = self.s.L.adfb_gmres_solve(2, b.ctypes.data, x.ctypes.data, b.size, restart, max_its, rtol, atol,
                                       C.cast(pc.fn, C.c_void_p) if pc else None, None, C.byref(its), C.byref(rn))
        check(rc, "adfb_gmres_solve")
        return x, its.value, rn.value

    def true_residual(self, b, x):
        """||b - T x|| in extended precision"""
        apply, _ = block_operator(self.T, None)
        return float(np.sqrt(np.sum((np.asarray(b, LD) - apply(np.asarray(x, LD))) ** 2)))


def system(key):
    if key not in _live:
        _drop()
        if key == "single":        # 9 x 8 x 7 cells, 5 unknowns each: n = 2520
            prm, hb = case(9, 8, 7)
            _live[key] = System(key, prm, SINGLE_ANK, [hb])
        elif key == "cell":        # one cell: n = 5
            prm, hb = case(1, 1, 1)
            _live[key] = System(key, prm, make_ank_params(cfl=3.0, coupled=False), [hb])
        elif key == "large":       # 40 x 32 x 16 cells, coupled: n = 122 880, the dots loop over the 256 CTAs
            prm, hb = case(40, 32, 16)
            ank = make_ank_params(cfl=3.0, coupled=True, char_time_step="VLR", cflLimit=20.0, turbCFLScale=2.0)
            _live[key] = System(key, prm, ank, [hb])
        elif key == "three":       # three blocks of different shapes: the dots reduce across blocks
            from test_multiblock_vectors import BlockSet

            bs = BlockSet(names=("B", "C", "D"))
            _live[key] = System(key, bs.prm, make_ank_params(cfl=3.0, coupled=False, char_time_step="Turkel"), bs.blocks)
    return _live[key]


# ---------------------------------------------------------------------------------------------------------------------
# checks
def check_iterate(sysm, b, ref, k, x, its, rn):
    bn = float(ref.bnorm)
    assert its == k
    check_x(sysm, x, ref.x[k], k)
    er = abs(rn - float(ref.res[k])) / bn
    assert er <= RES_TOL, ("resNorm", k, er)
    check_reported(sysm, b, x, rn)


def check_x(sysm, x, xk, what):
    xk = np.asarray(xk, dtype=np.float64)
    ex = np.linalg.norm(x - xk) / np.linalg.norm(xk)
    assert ex <= X_TOL[sysm.key], ("x", what, ex)


def check_reported(sysm, b, x, rn):
    """the reported residual is never below the true one by more than rounding"""
    true = sysm.true_residual(b, x)
    assert np.isfinite(true) and rn >= true - RES_TOL * np.linalg.norm(b), (rn, true)


def disc_case(sysm, seed, radius):
    rng = np.random.default_rng(seed)
    Minv = preconditioner_for(sysm.T, disc_spectrum(rng, sysm.nc, sysm.ns, radius))
    return Minv, rng.standard_normal(sysm.n)


# ---------------------------------------------------------------------------------------------------------------------
# every iterate
@pytest.mark.parametrize("restart", [1, 2, 7, 30, 60, 126])
def test_every_iterate(cuda_lib, restart):
    """x_k for every k of two restart cycles and the first step of the third (at least eight steps), eigenvalues filling
    the disc of radius 0.95 about 1: the residual falls by a factor of about 0.9 a step, so even a first cycle of 126
    steps ends far above rounding"""
    sysm = system("single")
    Minv, b = disc_case(sysm, restart, 0.95)
    kmax = max(2 * restart + 1, 8)
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, restart, kmax, minv=minv)
    assert float(ref.res[restart]) > 1e-9 * float(ref.bnorm)
    pc = Precond(Minv)
    for k in range(1, kmax + 1):
        x, its, rn = sysm.solve(b, restart, k, pc=pc)
        check_iterate(sysm, b, ref, k, x, its, rn)


def test_preconditioned_restarts(cuda_lib):
    """an inexact M^-1, the block inverse of the time-step matrix of a state perturbed by up to 5 %, over four cycles of
    5: the residual falls from 1 to about 1e-5"""
    sysm = system("single")
    prm, hb = case(9, 8, 7)
    rng = np.random.default_rng(17)
    ow = hb.d.owned()
    hb.w[ow] *= 1.0 + 0.05 * rng.uniform(-1.0, 1.0, hb.w[ow].shape)
    Minv = np.linalg.inv(time_step_blocks(prm, SINGLE_ANK, hb))
    b = rng.standard_normal(sysm.n)
    restart, kmax = 5, 20
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, restart, kmax, minv=minv)
    assert float(ref.res[kmax]) > 1e-9 * float(ref.bnorm)
    pc = Precond(Minv)
    for k in range(1, kmax + 1):
        x, its, rn = sysm.solve(b, restart, k, pc=pc)
        check_iterate(sysm, b, ref, k, x, its, rn)


# ---------------------------------------------------------------------------------------------------------------------
# stopping rules
@pytest.mark.parametrize("rule", ["rtol", "atol"])
def test_stopping_rules(cuda_lib, rule):
    """a target 5 % above the exact residual of step k and below that of step k - 1 stops the solve at k: inside the
    first cycle, exactly on the restart boundary (k = 7), on the first step of the second cycle (k = 8) and later"""
    sysm = system("single")
    Minv, b = disc_case(sysm, 3, 0.6)
    restart, kmax = 7, 16
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, restart, kmax, minv=minv)
    res = np.array(ref.res, dtype=np.float64)
    bn = float(ref.bnorm)
    pc = Precond(Minv)
    for k in (1, 3, 7, 8, 9, 15):
        assert res[k - 1] > 1.1 * res[k]                # the target lies well between the two
        target = 1.05 * res[k]
        rtol, atol = (target / bn, 0.0) if rule == "rtol" else (0.0, target)
        assert ref.first_k(rtol, atol) == k
        x, its, rn = sysm.solve(b, restart, 50, rtol=rtol, atol=atol, pc=pc)
        check_iterate(sysm, b, ref, k, x, its, rn)
        assert rn <= target
    # the larger of rtol ||b|| and atol decides
    x, its, rn = sysm.solve(b, restart, 50, rtol=1.05 * res[8] / bn, atol=1.05 * res[3], pc=pc)
    assert its == 3


def test_zero_and_small_right_hand_sides(cuda_lib):
    sysm = system("single")
    Minv, b = disc_case(sysm, 4, 0.9)
    pc = Precond(Minv)
    x, its, rn = sysm.solve(np.zeros(sysm.n), 7, 20, rtol=1e-6, pc=pc)
    assert its == 0 and rn == 0.0 and not np.any(x) and pc.calls == 0
    x, its, rn = sysm.solve(np.zeros(sysm.n), 7, 20, pc=pc)            # rtol = atol = 0 as well
    assert its == 0 and rn == 0.0 and not np.any(x) and pc.calls == 0
    bn = np.linalg.norm(b)
    for atol in (bn * (1 + 1e-12), 2.0 * bn):
        x, its, rn = sysm.solve(b, 7, 20, atol=atol, pc=pc)
        assert its == 0 and abs(rn - bn) <= 1e-14 * bn and not np.any(x) and pc.calls == 0


# ---------------------------------------------------------------------------------------------------------------------
# termination and saturation
def test_few_distinct_eigenvalues_terminate(cuda_lib):
    """four distinct eigenvalues: the residual vanishes (to rounding) at step 4 and not before"""
    sysm = system("single")
    rng = np.random.default_rng(21)
    Minv = preconditioner_for(sysm.T, few_values_spectrum(rng, sysm.nc, sysm.ns, [0.5, 1.0, 2.0, 3.5]))
    b = rng.standard_normal(sysm.n)
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, 30, 8, minv=minv)
    res = np.array(ref.res, dtype=np.float64) / float(ref.bnorm)
    assert np.all(res[:4] > 1e-3) and res[4] < 1e-13
    pc = Precond(Minv)
    for k in range(1, 5):
        x, its, rn = sysm.solve(b, 30, k, pc=pc)
        check_iterate(sysm, b, ref, k, x, its, rn)
    x, its, rn = sysm.solve(b, 30, 30, rtol=1e-10, pc=pc)
    assert its == 4 and rn <= 1e-10 * np.linalg.norm(b)
    check_reported(sysm, b, x, rn)


def test_invariant_right_hand_side(cuda_lib):
    """b an eigenvector of T M^-1 (the real eigenvalue of one cell): one step solves it"""
    sysm = system("single")
    rng = np.random.default_rng(5)
    nc, ns = sysm.nc, sysm.ns
    D = np.zeros((nc, ns, ns))
    D[:, np.arange(ns), np.arange(ns)] = rng.uniform(0.5, 2.0, (nc, ns))
    Q, _ = np.linalg.qr(rng.standard_normal((nc, ns, ns)))
    Minv = preconditioner_for(sysm.T, Q @ D @ np.transpose(Q, (0, 2, 1)))
    b = np.zeros(sysm.n)
    q = nc // 3
    b[q * ns:(q + 1) * ns] = 2.0 * Q[q][:, 2]
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, 30, 3, minv=minv)
    assert float(ref.res[1]) < 1e-14 * float(ref.bnorm)
    pc = Precond(Minv)
    x, its, rn = sysm.solve(b, 30, 30, rtol=1e-10, pc=pc)
    check_iterate(sysm, b, ref, 1, x, its, rn)


def test_restart_beyond_the_dimension(cuda_lib):
    """one cell, n = 5: GMRES(30) has the solution after 5 steps; the steps after it must not spoil x"""
    sysm = system("cell")
    assert sysm.n == 5
    Minv, b = disc_case(sysm, 8, 0.9)
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, 30, 30, minv=minv)
    assert float(ref.res[5]) < 1e-15 * float(ref.bnorm)
    pc = Precond(Minv)
    for k in range(1, 5):
        x, its, rn = sysm.solve(b, 30, k, pc=pc)
        check_iterate(sysm, b, ref, k, x, its, rn)
    xs = ref.x[5]
    for max_its in (5, 6, 12, 30, 61):
        x, its, rn = sysm.solve(b, 30, max_its, pc=pc)
        assert 5 <= its <= max_its
        check_x(sysm, x, xs, (max_its, its))
        check_reported(sysm, b, x, rn)


@pytest.mark.parametrize("key", ["large", "three"])
def test_large_and_several_blocks(cuda_lib, key):
    """n = 122 880 in one coupled block, and three blocks of different shapes: iterates inside and across restarts"""
    sysm = system(key)
    Minv, b = disc_case(sysm, 30, 0.9)
    restart, ks = 30, (1, 2, 17, 30, 31, 45)
    apply, minv = block_operator(sysm.T, Minv)
    ref = ExactGmres(apply, b, restart, max(ks), minv=minv)
    pc = Precond(Minv)
    for k in ks:
        x, its, rn = sysm.solve(b, restart, k, pc=pc)
        check_iterate(sysm, b, ref, k, x, its, rn)


# ---------------------------------------------------------------------------------------------------------------------
# breakdown and non-finite values
def test_zero_column(cuda_lib):
    """M^-1 with a null space (a zero block on a third of the cells) and b supported there: A M^-1 v_0 = 0, a zero
    column at the first step.  No Krylov vector can reduce the residual, so the solve ends after that step with x = 0
    and resNorm = ||b||, which no restart could change"""
    sysm = system("single")
    Minv, _ = disc_case(sysm, 9, 0.9)
    ns = sysm.ns
    null = np.arange(sysm.nc) % 3 == 1
    Minv[null] = 0.0
    b = np.zeros(sysm.n)
    b.reshape(-1, ns)[null] = np.random.default_rng(9).standard_normal((int(null.sum()), ns))
    b *= 2.0 / np.linalg.norm(b)
    pc = Precond(Minv)
    for restart, max_its in ((7, 20), (1, 5), (30, 1)):
        x, its, rn = sysm.solve(b, restart, max_its, rtol=1e-8, pc=pc)
        assert its == 1 and not np.any(x)
        assert abs(rn - 2.0) <= RES_TOL * 2.0, rn
        check_reported(sysm, b, x, rn)
    # b with a part outside the null space: that part is solved, the rest stays, and the residual never reads below it
    b2 = b + np.where(np.repeat(null, ns), 0.0, 1.0) * np.random.default_rng(10).standard_normal(sysm.n)
    x, its, rn = sysm.solve(b2, 7, 60, rtol=1e-8, pc=pc)
    check_reported(sysm, b2, x, rn)
    assert rn >= 2.0 * (1 - 1e-12)


@pytest.mark.parametrize("restart,max_its", [(7, 20), (2, 20), (2, 2)])
def test_nan_from_the_preconditioner(cuda_lib, restart, max_its):
    """a NaN from the callback's third call: inside the first cycle (restart 7), in the update that closes it (restart 2),
    and that update as the last step (maxIts 2).  The solve stops with resNorm NaN and returns 0"""
    sysm = system("single")
    Minv, b = disc_case(sysm, 11, 0.9)
    pc = Precond(Minv, nan_at=3)
    x, its, rn = sysm.solve(b, restart, max_its, rtol=1e-10, pc=pc)
    assert np.isnan(rn), (its, rn)
    assert 1 <= its <= 3 and pc.calls == 3, (its, pc.calls)


def test_non_finite_right_hand_side(cuda_lib):
    sysm = system("single")
    Minv, b = disc_case(sysm, 12, 0.9)
    for bad in (np.nan, np.inf):
        bb = b.copy()
        bb[17] = bad
        pc = Precond(Minv)
        x, its, rn = sysm.solve(bb, 7, 20, rtol=1e-8, atol=1e-30, pc=pc)
        assert np.isnan(rn) and its == 0 and pc.calls == 0 and not np.any(x)
