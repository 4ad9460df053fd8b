"""The exact iterates of right-preconditioned restarted GMRES(m) with a zero initial guess, for the device GMRES
(adfb_gmres_solve) to be measured against.

The iterates are defined by the mathematics, not by an algorithm.  With A the preconditioned operator T M^-1:
  - in the first cycle, y_k minimises ||b - A y|| over y in K_k(A, b) and x_k = M^-1 y_k;
  - after each restart (every m steps), the same holds from the true residual r = b - A y_m of the restart point.
They are computed here by Arnoldi with full reorthogonalisation (classical Gram-Schmidt run twice) and a Givens
least-squares solve, all in extended precision (np.longdouble, 64-bit mantissa), and every residual is formed again
from its iterate, ||b - A y_k||, not taken from the recurrence.  T and M^-1 are taken as the exact doubles they hold.
tests/test_gmres_ref_host.py checks this against mpmath at 50 digits and against closed forms."""
import numpy as np

LD = np.longdouble
assert np.finfo(LD).eps <= 1.1e-19, "the exact GMRES reference needs an extended-precision np.longdouble"


def block_operator(T, Minv):
    """(apply, minv) of the block-diagonal operator T M^-1 in extended precision: T and Minv are (ncells, ns, ns) arrays of
    doubles (Minv None: the identity), vectors cell-major like the library's state vectors"""
    TL = np.asarray(T, dtype=LD)
    ns = TL.shape[1]
    ML = None if Minv is None else np.asarray(Minv, dtype=LD)

    def minv(v):
        return v if ML is None else np.einsum("qlm,qm->ql", ML, v.reshape(-1, ns)).reshape(-1)

    def apply(v):
        return np.einsum("qlm,qm->ql", TL, minv(v).reshape(-1, ns)).reshape(-1)

    return apply, minv


def _norm(v):
    return np.sqrt(np.dot(v, v))


class ExactGmres:
    """GMRES(restart) iterates k = 0 .. kmax of A y = b (x = M^-1 y) in extended precision.

    apply: the preconditioned operator A = T M^-1 on longdouble vectors; minv: M^-1 (None: identity).
    x[k] (longdouble), res[k] = ||b - A y_k||, bnorm = ||b||.  An iterate whose Krylov space is invariant (a happy
    breakdown, the new Arnoldi vector below `breakdown` times the product it came from) is the exact solution; every
    later iterate equals it."""

    def __init__(self, apply, b, restart, kmax, minv=None, breakdown=1e-15):
        minv = minv or (lambda v: v)
        b = np.asarray(b, dtype=LD)
        n, m = b.size, restart
        self.bnorm = _norm(b)
        y = np.zeros(n, dtype=LD)
        self.x, self.res = [minv(y)], [self.bnorm]
        done = self.bnorm == 0
        while len(self.res) <= kmax and not done:
            r = b - apply(y)
            beta = _norm(r)
            if beta == 0:
                break
            V = np.zeros((m + 1, n), dtype=LD)
            V[0] = r / beta
            R = np.zeros((m + 1, m), dtype=LD)          # the triangular factor of the Hessenberg matrix
            cs, sn = np.zeros(m, dtype=LD), np.zeros(m, dtype=LD)
            g = np.zeros(m + 1, dtype=LD)
            g[0] = beta
            yk = y
            for j in range(m):
                w = apply(V[j])
                wn = _norm(w)
                h = np.zeros(j + 2, dtype=LD)
                for _ in range(2):
                    c = V[:j + 1] @ w
                    w = w - c @ V[:j + 1]
                    h[:j + 1] += c
                h[j + 1] = _norm(w)
                for i in range(j):
                    h[i], h[i + 1] = cs[i] * h[i] + sn[i] * h[i + 1], -sn[i] * h[i] + cs[i] * h[i + 1]
                den = np.hypot(h[j], h[j + 1])
                if den == 0:                                # A v_j in the span of A v_0 .. A v_j-1: no progress, ever
                    done = True
                    self.x.append(self.x[-1])
                    self.res.append(self.res[-1])
                    break
                cs[j], sn[j] = h[j] / den, h[j + 1] / den
                h[j], h[j + 1] = den, 0
                g[j], g[j + 1] = cs[j] * g[j], -sn[j] * g[j]
                R[:j + 1, j] = h[:j + 1]
                c = np.zeros(j + 1, dtype=LD)
                for i in range(j, -1, -1):
                    c[i] = (g[i] - R[i, i + 1:j + 1] @ c[i + 1:]) / R[i, i]
                yk = y + c @ V[:j + 1]
                self.x.append(minv(yk))
                self.res.append(_norm(b - apply(yk)))
                if len(self.res) > kmax:
                    break
                hn = _norm(w)
                if hn <= breakdown * wn:
                    done = True
                    break
                V[j + 1] = w / hn
            y = yk
        while len(self.res) <= kmax:
            self.x.append(self.x[-1])
            self.res.append(self.res[-1])

    def first_k(self, rtol, atol):
        """the first k whose residual meets max(rtol ||b||, atol), None if no k <= kmax does"""
        target = max(LD(rtol) * self.bnorm, LD(atol))
        for k, r in enumerate(self.res):
            if r <= target:
                return k
        return None
