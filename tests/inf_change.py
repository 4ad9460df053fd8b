"""infChangeCorrection and setUniformFlow (src/initFlow/initializeFlow.F90:191-316, :2143-2212) restated on oracle blocks,
in the reference's operation order, for the tests.

infChangeCorrection, with the new free stream wInf of the parameters and the old one oldWinf(1:5):

  deltaWinf = wInf(1:5) - oldWinf
  return if myNorm2(deltaWinf) < tol           myNorm2 (utils.F90:1696-1702) has a dimension(3) dummy: rho, u, v only
  "offset": w(2:il, 2:jl, 2:kl, 1:5) += deltaWinf
  "rotate": v <- ((r1 v1 + r2 v2) + r3 v3) * mag2 / mag1 per row of rotMat = getRotMatrix(old, new velocity)
            (utils.F90:6591-6665), rho and rhoE += their offsets
  then per block applyAllBC_block(.true.) (flow BCs, second halos, the pressure NOT recomputed first), whalo2(1, 1, nw,
  T, T, T) (exchange, orphan averaging, computeEtotBlock on the owned cells), and with overset blocks the turbulence and
  flow BCs once more.

Elementwise numpy arithmetic rounds every operation, as the reference (and the device, with explicit roundings) does.
The exchange is the caller's: a function of the list of blocks (the numpy model of adflow_b200.halo), or None."""
import ctypes as C
import ctypes.util
import math

import numpy as np

_M = C.CDLL(ctypes.util.find_library("m"))
for _f in ("acos", "sin", "cos", "sqrt"):
    getattr(_M, _f).restype = C.c_double
    getattr(_M, _f).argtypes = [C.c_double]

KINDS = ("offset", "rotate")


def options(eq, lift=2):
    return {"equationType": eq, "liftIndex": lift}


def with_free_stream(prm, mach, alpha_deg, lift, p_ratio=1.0, t_ratio=1.0):
    """a copy of prm whose free stream (pInf, pInfCorr, rhoInf, wInf(1:5)) is that of a new AeroProblem: Mach number, alpha
    (about the axis of liftIndex), pressure and temperature relative to those of prm, which fixed the reference state.
    With the same values it reproduces make_params' free stream bit for bit.  The turbulence entry is kept: the
    correction does not touch it."""
    from adflow_b200.params import AdfbParams

    q = AdfbParams.from_buffer_copy(prm)
    q._muInf = prm._muInf
    gamma = prm.gammaInf
    p, rho = p_ratio, p_ratio / t_ratio
    u = mach * math.sqrt(gamma * p / rho)
    a = math.radians(alpha_deg)
    vdir = (math.cos(a), math.sin(a), 0.0) if lift == 2 else (math.cos(a), 0.0, math.sin(a))
    q.wInf[0], q.wInf[1], q.wInf[2], q.wInf[3] = rho, u * vdir[0], u * vdir[1], u * vdir[2]
    q.wInf[4] = rho * (p / ((gamma - 1.0) * rho) + 0.5 * u * u)
    q.pInf = q.pInfCorr = p
    q.rhoInf = rho
    return q


def free_stream_pair(eq, change, lift=2):
    """(old, new) parameters of one AeroProblem change from Mach 0.8, alpha 1.8"""
    from adflow_b200 import make_params

    prm0 = make_params(options(eq, lift))
    new = {"alpha": (0.8, 2.8, 1.0, 1.0), "mach": (0.75, 1.8, 1.0, 1.0), "pressure": (0.8, 1.8, 1.1, 1.0),
           "temperature": (0.8, 1.8, 1.0, 0.95)}[change]
    return prm0, with_free_stream(prm0, new[0], new[1], lift, new[2], new[3])


def sign_flip_pair(eq):
    """alpha +2 -> -2 degrees with liftIndex 3: only w and nothing of rho, u, v changes, so the reference skips it"""
    from adflow_b200 import make_params

    prm0 = make_params(options(eq, 3), alpha_deg=2.0)
    return prm0, with_free_stream(prm0, 0.8, -2.0, 3)


def my_norm2(x):
    """myNorm2: sqrt(x(1)**2 + x(2)**2 + x(3)**2) of the first three entries"""
    return _M.sqrt(x[0] * x[0] + x[1] * x[1] + x[2] * x[2])


def rot_matrix(vec1, vec2):
    """getRotMatrix: Rodrigues' formula, matmul sums from zero in index order; rotMat as a 3 x 3 nested list"""
    f = np.float64   # numpy scalars: 0 / 0 is NaN, as in the reference, not an exception
    v1, v2 = [f(v) for v in vec1], [f(v) for v in vec2]
    with np.errstate(all="ignore"):
        dot = f(0.0)
        for i in range(3):
            dot = dot + v1[i] * v2[i]
        cosine = dot / (f(my_norm2(v1)) * f(my_norm2(v2)))
        theta = _M.acos(cosine)
        v3 = [v1[1] * v2[2] - v1[2] * v2[1], v1[2] * v2[0] - v1[0] * v2[2], v1[0] * v2[1] - v1[1] * v2[0]]
        ln = f(_M.sqrt(v3[0] * v3[0] + v3[1] * v3[1] + v3[2] * v3[2]))
        v3 = [v / ln for v in v3]
        W = [[f(0.0), -v3[2], v3[1]], [v3[2], f(0.0), -v3[0]], [-v3[1], v3[0], f(0.0)]]
        s, c = f(_M.sin(theta)), f(1.0 - _M.cos(theta))
        rot = [[0.0] * 3 for _ in range(3)]
        for i in range(3):
            for j in range(3):
                w2 = f(0.0)
                for k in range(3):
                    w2 = w2 + W[i][k] * W[k][j]
                rot[i][j] = float((f(1.0 if i == j else 0.0) + s * W[i][j]) + c * w2)
    return rot


def delta_winf(prm, old_winf):
    return [prm.wInf[l] - float(old_winf[l]) for l in range(5)]


def skipped(prm, old_winf, tol):
    """the reference's early return"""
    return my_norm2(delta_winf(prm, old_winf)) < tol


def correct_owned(hb, prm, old_winf, kind):
    """the update of the owned cells of one level-1 block"""
    dwinf = delta_winf(prm, old_winf)
    ow = hb.d.owned()
    w = hb.w
    if kind == "offset":
        for l in range(5):
            w[ow + (l,)] = w[ow + (l,)] + dwinf[l]
        return
    old_v, new_v = [float(old_winf[l]) for l in (1, 2, 3)], [prm.wInf[l] for l in (1, 2, 3)]
    rot = rot_matrix(old_v, new_v)
    mag1, mag2 = my_norm2(old_v), my_norm2(new_v)
    v = [w[ow + (l,)].copy() for l in (1, 2, 3)]
    with np.errstate(all="ignore"):
        for m in range(3):
            r = (rot[m][0] * v[0] + rot[m][1] * v[1]) + rot[m][2] * v[2]
            w[ow + (m + 1,)] = r * mag2 / mag1
    w[ow + (0,)] = w[ow + (0,)] + dwinf[0]
    w[ow + (4,)] = w[ow + (4,)] + dwinf[4]


def inf_change_correction(blocks, prm, old_winf, tol=1e-12, kind="offset", exchange=None, overset=False):
    """the whole routine on the level-1 blocks (in place); returns whether it changed anything"""
    from oracle.pyoracle import Oracle

    if skipped(prm, old_winf, tol):
        return False
    for hb in blocks:
        correct_owned(hb, prm, old_winf, kind)
        Oracle(hb, prm).apply_flow_bc(True)
    if exchange is not None:
        exchange(blocks)
    for hb in blocks:   # whalo2's computeEtotBlock(2, il, 2, jl, 2, kl)
        d = hb.d
        o = Oracle(hb, prm)
        o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    if overset:
        for hb in blocks:
            o = Oracle(hb, prm)
            if prm.equations == 3:
                o.apply_turb_bc(True)
            o.apply_flow_bc(True)
    return True


def set_uniform_flow(hb, prm, mu_inf, eddy_vis_inf_ratio):
    """setUniformFlow on one block (in place), halos included"""
    hb.w[...] = np.asarray(prm.wInf[:hb.nw])
    hb.dw[...] = 0.0
    hb.fw[...] = 0.0
    hb.p[...] = prm.pInfCorr
    if prm.equations != 1:
        hb.rlv[...] = mu_inf
    if prm.equations == 3:
        hb.rev[...] = eddy_vis_inf_ratio * mu_inf
