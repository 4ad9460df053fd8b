"""The exact GMRES reference (tests/gmres_ref.py) against mpmath at 50 digits and against closed forms.

The mpmath iterates come from the definition alone: y_k minimises ||r0 - A y|| over the span of the Krylov matrix
[r0, A r0, .., A^(k-1) r0], solved by the normal equations at 50 digits, with no Arnoldi process and no rotation."""
import mpmath
import numpy as np
import pytest

from gmres_ref import LD, ExactGmres, block_operator

mp = mpmath.mp


def _ld_dense(A):
    AL = np.asarray(A, dtype=LD)
    return lambda v: AL @ v


def mp_gmres(A, Minv, b, restart, kmax):
    """x_k and ||b - A y_k|| of GMRES(restart) by the definition; A = T M^-1 (an mpmath matrix or doubles)"""
    with mp.workdps(50):
        Am = A if isinstance(A, mp.matrix) else mp.matrix(A.tolist())
        Mm, bm = mp.matrix(Minv.tolist()), mp.matrix(b.tolist())
        n = len(b)
        y = mp.matrix(n, 1)
        xs, res = [Mm * y], [mp.norm(bm)]
        while len(res) <= kmax:
            r0 = bm - Am * y
            K = mp.matrix(n, restart)
            v = r0
            for j in range(restart):
                K[:, j] = v
                v = Am * v
            for k in range(1, restart + 1):
                AK = Am * K[:, :k]
                c = mp.lu_solve(AK.T * AK, AK.T * r0)
                yk = y + K[:, :k] * c
                xs.append(Mm * yk)
                res.append(mp.norm(bm - Am * yk))
                if len(res) > kmax:
                    break
            y = yk
        return [np.array([float(t) for t in xk]) for xk in xs], np.array([float(t) for t in res])


def _check_against_mp(ref, xs, res, tol):
    for k, (xk, rk) in enumerate(zip(xs, res)):
        xl = np.asarray(ref.x[k], dtype=np.float64)
        assert np.linalg.norm(xl - xk) <= tol * max(np.linalg.norm(xk), 1e-300), k
        assert abs(float(ref.res[k]) - rk) <= tol * float(ref.bnorm), k


@pytest.mark.parametrize("n,restart,kmax", [(12, 4, 11), (9, 1, 6), (10, 3, 10)])
def test_dense_operator_against_mpmath(n, restart, kmax):
    rng = np.random.default_rng(n * 31 + restart)
    A = np.eye(n) * 2.0 + rng.standard_normal((n, n)) * 0.4
    Minv = np.eye(n) + rng.standard_normal((n, n)) * 0.1
    b = rng.standard_normal(n)
    ref = ExactGmres(_ld_dense(A), b, restart, kmax, minv=_ld_dense(Minv))
    xs, res = mp_gmres(A, Minv, b, restart, kmax)
    # residuals fall from 1 to about 1e-3 here: well inside what double precision could still tell apart
    assert res[-1] < 0.5 * res[0] and np.all(np.diff(res) <= 1e-15)
    _check_against_mp(ref, xs, res, 1e-15)


def test_block_operator_against_mpmath():
    """T M^-1 block by block (3 cells of 5 unknowns): the layout the device vectors have"""
    rng = np.random.default_rng(7)
    nc, ns = 3, 5
    T = np.eye(ns) * 3.0 + rng.standard_normal((nc, ns, ns))
    Minv = np.linalg.inv(T) @ (np.eye(ns) + 0.5 * rng.standard_normal((nc, ns, ns)))
    b = rng.standard_normal(nc * ns)
    apply, minv = block_operator(T, Minv)
    ref = ExactGmres(apply, b, 6, 14, minv=minv)
    n = nc * ns
    Td, Md = np.zeros((n, n)), np.zeros((n, n))
    for q in range(nc):
        Td[q * ns:(q + 1) * ns, q * ns:(q + 1) * ns] = T[q]
        Md[q * ns:(q + 1) * ns, q * ns:(q + 1) * ns] = Minv[q]
    with mp.workdps(50):
        A = mp.matrix(Td.tolist()) * mp.matrix(Md.tolist())
    xs, res = mp_gmres(A, Md, b, 6, 14)
    _check_against_mp(ref, xs, res, 1e-14)
    assert res[14] < 0.2 * res[0]


def test_distinct_eigenvalues_terminate():
    """a diagonal operator with d distinct values: the minimal polynomial has degree d, so y_d is the solution and no
    earlier iterate is"""
    d, n = 7, 40
    vals = np.array([0.5, 1.0, 1.7, 2.5, -1.3, 4.0, 9.0])
    diag = np.resize(vals, n)
    b = np.random.default_rng(3).standard_normal(n)
    ref = ExactGmres(lambda v: np.asarray(diag, dtype=LD) * v, b, 20, 12)
    res = np.array(ref.res, dtype=np.float64)
    assert np.all(res[:d] > 1e-3 * res[0]) and np.all(np.diff(res[:d]) < 0)
    assert res[d] < 1e-16 * res[0]          # double precision cannot tell it from zero
    assert np.allclose(np.asarray(ref.x[d], dtype=np.float64), b / diag, rtol=1e-15, atol=0)
    assert all(ref.x[k] is ref.x[d] for k in range(d + 1, 13))


def test_gmres1_is_minimal_residual_step_by_step():
    """GMRES(1): x_k+1 = x_k + a r_k with a = (r_k, A r_k) / (A r_k, A r_k), the minimal residual iteration"""
    rng = np.random.default_rng(11)
    n = 8
    A = np.eye(n) * 2.0 + rng.standard_normal((n, n)) * 0.3
    b = rng.standard_normal(n)
    ref = ExactGmres(_ld_dense(A), b, 1, 10)
    with mp.workdps(40):
        Am, bm = mp.matrix(A.tolist()), mp.matrix(b.tolist())
        x = mp.matrix(n, 1)
        for k in range(1, 11):
            r = bm - Am * x
            Ar = Am * r
            x = x + r * (mp.fdot(r, Ar) / mp.fdot(Ar, Ar))
            xk = np.array([float(t) for t in x])
            assert np.linalg.norm(np.asarray(ref.x[k], dtype=np.float64) - xk) <= 1e-16 * np.linalg.norm(xk), k
            assert abs(float(ref.res[k]) - float(mp.norm(bm - Am * x))) <= 1e-16 * float(ref.bnorm), k


def test_first_k_and_trivial_right_hand_sides():
    rng = np.random.default_rng(5)
    n = 30
    A = np.diag(np.linspace(1.0, 20.0, n))
    b = rng.standard_normal(n)
    ref = ExactGmres(_ld_dense(A), b, 5, 12)
    res = np.array(ref.res, dtype=np.float64)
    bn = float(ref.bnorm)
    for k in range(1, 13):
        assert ref.first_k(res[k] * 1.05 / bn, 0.0) == k
        assert ref.first_k(0.0, res[k] * 1.05) == k
        assert ref.first_k(res[k] * 1.05 / bn, res[k] * 0.5) == k      # the larger of the two decides
    assert ref.first_k(res[12] * 0.5 / bn, 0.0) is None
    assert ref.first_k(0.0, bn * 1.01) == 0
    z = ExactGmres(_ld_dense(A), np.zeros(n), 5, 4)
    assert z.first_k(0.0, 0.0) == 0 and all(float(r) == 0.0 for r in z.res) and not np.any(np.asarray(z.x[4], dtype=float))
