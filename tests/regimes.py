"""Flow regimes the smooth synthetic state never reaches, and numpy measures of which branches they reach.

``synthetic.fill_state`` is a subsonic free stream with a 5 % smooth perturbation: the JST sensor stays near 1e-3, no
far-field face is supersonic and no floor is hit, so every branch the kernels take *from the state* runs on one side
only.  ``regime_case`` builds blocks that reach the other side:

  contact_i / contact_j / contact_k   density x 1/8 at constant pressure across one plane of one index direction
                                      (entropy x 18): sensor cap min(0.25, dss) and dis4 = 0 on that direction's faces
  contact_pocket                      density x 1/8 at constant pressure in a 4^3 cube of interior cells: the sensor cap
                                      on faces of all three directions in a state that stays bounded over smoother cycles
  supersonic                          M 2.0, alpha 20 deg free stream with a pocket of density x 1/8, pressure x 2
                                      (locally subsonic): both supersonic far-field branches, one-signed eigenvalues,
                                      entropy and pressure sensor caps
  stagnation                          a j slab with |u| x 1e-3 and nuTilde x 100: near-zero normal velocities, SA rr clip
  floors                              one plane whose internal energy lies below the pressure floor 1e-4 pInfCorr and
                                      nuTilde below the setW clip 1e-6 nuInf in the cells of another plane
  low_mach                            M 0.3, alpha 25 deg, far field on both j faces: far-field inflow and outflow on j

A contact that spans the block (contact_i/j/k) puts the low-density side against the far-field faces; an explicit
smoother cycle on it diverges within one cycle in the reference's own executeRKStage as much as in the oracle (the two
agree bit for bit), so the smoother tests use contact_pocket.

``reach`` counts, from the input state alone, how often each branch is taken, so that a test can assert that its
regime still reaches the branches it is meant to exercise before it compares anything.
"""
import math

import numpy as np

from adflow_b200 import make_params
from adflow_b200 import synthetic as syn
from adflow_b200.params import EULER, RANS

REGIMES = ("contact_i", "contact_j", "contact_k", "contact_pocket", "supersonic", "stagnation", "floors", "low_mach")
FREE_STREAM = {"supersonic": (2.0, 20.0), "low_mach": (0.3, 25.0)}   # (Mach, alpha in degrees); M 0.8 / 1.8 deg otherwise
LOW_MACH_FACES = {syn.IMIN: syn.BC_FARFIELD, syn.IMAX: syn.BC_FARFIELD, syn.JMIN: syn.BC_FARFIELD,
                  syn.JMAX: syn.BC_FARFIELD, syn.KMIN: syn.BC_WALL, syn.KMAX: syn.BC_FARFIELD}
DENSITY_JUMP = 1.0 / 8.0
PRESSURE_FLOOR = 1e-4          # x pInfCorr: state preparation and the Runge-Kutta update
TURB_CLIP = 1e-6               # x wInf[5]: setW


def _refresh(prm, hb, p=None):
    """rhoE from p (or p from rhoE when p is None, floored like the state preparation), then rlv and rev -- the
    same relations fill_state uses, over the whole box"""
    w, gam = hb.w, prm.gammaInf
    v2 = w[..., 1] ** 2 + w[..., 2] ** 2 + w[..., 3] ** 2
    if p is None:
        p = np.maximum((gam - 1.0) * (w[..., 4] - 0.5 * w[..., 0] * v2), PRESSURE_FLOOR * prm.pInfCorr)
    else:
        w[..., 4] = p / (gam - 1.0) + 0.5 * w[..., 0] * v2
    hb.p[...] = p
    if prm.equations != EULER:
        hb.rlv[...] = syn.lam_viscosity(prm, hb.p, w[..., 0])
    if prm.equations == RANS:
        hb.rev[...] = syn.eddy_viscosity(prm, w, hb.rlv)


def contact_plane(name, shape):
    """default first cell (box index) on the far side of the discontinuity: the mid plane of the regime's direction"""
    a = "ijk".index(name[-1])
    return 2 + shape[a] // 2


def regime_case(name, shape, options=None, at=None, seed=314):
    """(prm, hb) of regime `name` on a block of `shape` owned cells.  `at`: for the contact regimes, the first cell (box
    index, owned cells are 2..n+1) of the low-density side; the jump lies on the face between at-1 and at."""
    if name not in REGIMES:
        raise KeyError(name)
    mach, alpha = FREE_STREAM.get(name, (0.8, 1.8))
    prm = make_params(options, mach=mach, alpha_deg=alpha)
    kw = {"physical_faces": LOW_MACH_FACES} if name == "low_mach" else {}
    hb = syn.make_block(*shape, prm, seed=seed, **kw)
    d, w = hb.d, hb.w
    p = hb.p.copy()
    if name == "contact_pocket":
        ci, cj, ck = (2 + n // 2 for n in shape)
        w[ci - 2:ci + 2, cj - 2:cj + 2, ck - 2:ck + 2, 0] *= DENSITY_JUMP
    elif name.startswith("contact"):
        a = "ijk".index(name[-1])
        c0 = contact_plane(name, shape) if at is None else at
        sl = [slice(None)] * 3
        sl[a] = slice(c0, None)                     # halos included: the far side is low density up to the boundary
        w[tuple(sl) + (0,)] *= DENSITY_JUMP
    elif name == "supersonic":
        ci, cj, ck = (2 + n // 2 for n in shape)
        pocket = (slice(ci - 2, ci + 2), slice(cj - 2, cj + 2), slice(max(ck - 2, 2), ck + 2))
        w[pocket + (0,)] *= DENSITY_JUMP            # with p x 2 the sound speed is x 4: the pocket is subsonic
        p[pocket] *= 2.0                            # and the pressure sensor of matrix dissipation is capped too
    elif name == "stagnation":
        cj = 2 + shape[1] // 2
        slab = (slice(None), slice(cj - 1, cj + 2), slice(None))
        w[slab + (slice(1, 4),)] *= 1e-3
        if hb.nw > 5:
            w[slab + (5,)] *= 100.0
    elif name == "floors":
        ci = 2 + shape[0] // 2
        plane = (slice(ci, ci + 1), slice(2, d.jl + 1), slice(2, d.kl + 1))
        v2 = w[plane + (1,)] ** 2 + w[plane + (2,)] ** 2 + w[plane + (3,)] ** 2
        w[plane + (4,)] = 0.5 * w[plane + (0,)] * v2 + 1e-6 * prm.pInfCorr / (prm.gammaInf - 1.0)
        if hb.nw > 5:
            cj = 2 + shape[1] // 2
            w[2:d.il + 1, cj, 2:d.kl + 1, 5] = 1e-2 * TURB_CLIP * prm.wInf[5]
        _refresh(prm, hb, None)
        return prm, hb
    _refresh(prm, hb, p)
    return prm, hb


# ---------------------------------------------------------------------------------------------------------------------
# reach measures (numpy, from the input state)
def entropy_sensor(prm, hb):
    """dss(1:ie, 1:je, 1:ke, 3) of inviscidDissFluxScalar (blockette.F90:3055-3105): |second difference / sum| of the
    entropy p / rho**gamma (of p for Euler), floored by sslim; zero outside 1..ie"""
    gam = prm.gammaInf
    if prm.equations == EULER:
        ss, sslim = hb.p, 0.001 * prm.pInfCorr
    else:
        ss, sslim = hb.p / hb.w[..., 0] ** gam, 0.001 * prm.pInfCorr / prm.rhoInf ** gam
    d = hb.d
    dss = np.zeros(d.box + (3,))
    c = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    for a in range(3):
        lo, hi = list(c), list(c)
        lo[a] = slice(0, (d.ie, d.je, d.ke)[a])
        hi[a] = slice(2, (d.ib, d.jb, d.kb)[a] + 1)
        sm, sp, s0 = ss[tuple(lo)], ss[tuple(hi)], ss[c]
        dss[c + (a,)] = np.abs((sp - 2.0 * s0 + sm) / (sp + 2.0 * s0 + sm + sslim))
    return dss


def face_sensor(prm, hb, a, dss=None):
    """max(dss(c), dss(c+1)) on the faces 1..l of direction a and the owned rows 2..l of the others: what dmin(0.25, .)
    is applied to; `dss` defaults to the entropy sensor"""
    d = hb.d
    dss = (entropy_sensor(prm, hb) if dss is None else dss)[..., a]
    ls = (d.il, d.jl, d.kl)
    sl_m, sl_p = [], []
    for b in range(3):
        if b == a:
            sl_m.append(slice(1, ls[b] + 1)); sl_p.append(slice(2, ls[b] + 2))
        else:
            sl_m.append(slice(2, ls[b] + 1)); sl_p.append(slice(2, ls[b] + 1))
    return np.maximum(dss[tuple(sl_m)], dss[tuple(sl_p)])


def pressure_sensor(prm, hb):
    """dss of the matrix dissipation (blockette.F90:2515-2560): pressure second difference over a blend of the sum and
    the absolute first differences (omega 0.5), floored by plim = 0.001 pInfCorr; cells 1..ie"""
    d, p = hb.d, hb.p
    dss = np.zeros(d.box + (3,))
    c = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    for a in range(3):
        lo, hi = list(c), list(c)
        lo[a] = slice(0, (d.ie, d.je, d.ke)[a])
        hi[a] = slice(2, (d.ib, d.jb, d.kb)[a] + 1)
        pm, pp, p0 = p[tuple(lo)], p[tuple(hi)], p[c]
        dss[c + (a,)] = np.abs((pp - 2.0 * p0 + pm) / (0.5 * (pp + 2.0 * p0 + pm) + 0.5 * (np.abs(pp - p0) + np.abs(p0 - pm))
                                                      + 0.001 * prm.pInfCorr))
    return dss


def _normal_mach(prm, hb, a):
    """|u . n| / c at the owned cells, n the unit normal of the direction-a faces"""
    d = hb.d
    s = (hb.si, hb.sj, hb.sk)[a][d.owned()]
    n = s / np.linalg.norm(s, axis=-1)[..., None]
    w = hb.w[d.owned()]
    vn = (w[..., 1:4] * n).sum(-1)
    c = np.sqrt(prm.gammaInf * hb.p[d.owned()] / w[..., 0])
    return np.abs(vn) / c


def farfield_branches(prm, hb):
    """far-field faces per branch of bcFarfield (BCRoutines.F90:1282-1396) with rface = 0: vn0 = wInf . n against
    +-c0s, and the side the interior entropy is taken from"""
    c0s = math.sqrt(prm.gammaInf * prm.pInfCorr / prm.rhoInf)
    out = {"ff_sup_in": 0, "ff_sub_in": 0, "ff_sub_out": 0, "ff_sup_out": 0}
    byface = {}
    for s in hb.subfaces:
        if s["bcType"] != syn.BC_FARFIELD:
            continue
        vn0 = s["norm"][..., 0] * prm.wInf[1] + s["norm"][..., 1] * prm.wInf[2] + s["norm"][..., 2] * prm.wInf[3]
        cnt = {"ff_sup_in": int((vn0 <= -c0s).sum()), "ff_sub_in": int(((vn0 > -c0s) & (vn0 <= 0.0)).sum()),
               "ff_sub_out": int(((vn0 > 0.0) & (vn0 <= c0s)).sum()), "ff_sup_out": int((vn0 > c0s).sum())}
        byface[s["faceId"]] = cnt
        for k, v in cnt.items():
            out[k] += v
    return out, byface


def sa_rr_unclipped(prm, hb):
    """rr = nuTilde / (S~ kappa^2 d^2) of saSource (blockette.F90:976-1168, strain production) before min(rr, 10), owned
    cells"""
    d, w = hb.d, hb.w
    ow = d.owned()
    I, J, K = ow
    Im, Jm, Km = (slice(s.start - 1, s.stop - 1) for s in ow)
    Ip, Jp, Kp = (slice(s.start + 1, s.stop + 1) for s in ow)
    gv = np.zeros((3, 3) + (d.nx, d.ny, d.nz))
    for v in range(3):
        q = w[..., 1 + v]
        for m in range(3):
            gv[v, m] = (q[Ip, J, K] * hb.si[I, J, K, m] - q[Im, J, K] * hb.si[Im, J, K, m]
                        + q[I, Jp, K] * hb.sj[I, J, K, m] - q[I, Jm, K] * hb.sj[I, Jm, K, m]
                        + q[I, J, Kp] * hb.sk[I, J, K, m] - q[I, J, Km] * hb.sk[I, J, Km, m])
    fact = 0.25 / hb.vol[ow]
    sxx, syy, szz = 2 * fact * gv[0, 0], 2 * fact * gv[1, 1], 2 * fact * gv[2, 2]
    sxy, sxz, syz = fact * (gv[0, 1] + gv[1, 0]), fact * (gv[0, 2] + gv[2, 0]), fact * (gv[1, 2] + gv[2, 1])
    div2 = (2.0 / 3.0) * (sxx + syy + szz) ** 2
    strain2 = 2 * (sxy ** 2 + sxz ** 2 + syz ** 2) + sxx ** 2 + syy ** 2 + szz ** 2
    sqrt_prod = np.sqrt(np.maximum(2 * strain2 - div2, 1e-25))
    nt = w[ow + (5,)]
    nu = hb.rlv[ow] / w[ow + (0,)]
    chi = nt / nu
    fv1 = chi ** 3 / (chi ** 3 + prm.rsaCv1 ** 3)
    fv2 = 1.0 - chi / (1.0 + chi * fv1)
    k2i = 1.0 / prm.rsaK ** 2
    d2i = 1.0 / hb.d2Wall[ow] ** 2
    sst = np.maximum(sqrt_prod + nt * fv2 * k2i * d2i, 1e-10)
    return nt * k2i * d2i / sst


def reach(prm, hb, regime=None):
    """branch counts of the input state (numpy only; `regime` is informational)"""
    d = hb.d
    ow = d.owned()
    r = {}
    for a, nm in enumerate("ijk"):
        fs = face_sensor(prm, hb, a)
        r["sensor_cap_" + nm] = int((fs >= 0.25).sum())          # dis2 = fis2 rrad 0.25
        # dis4 = max(fis4 rrad - dis2, 0) = 0 where fis2 min(0.25, dss) >= fis4
        r["dis4_zero_" + nm] = int((prm.vis2 * np.minimum(0.25, fs) >= prm.vis4).sum())
        r["matrix_sensor_cap_" + nm] = int((face_sensor(prm, hb, a, pressure_sensor(prm, hb)) >= 0.25).sum())
        r["supersonic_" + nm] = int((_normal_mach(prm, hb, a) > 1.0).sum())
        r["stagnant_" + nm] = int((_normal_mach(prm, hb, a) < 1e-2).sum())
    ff, _ = farfield_branches(prm, hb)
    r.update(ff)
    gam = prm.gammaInf
    w = hb.w[ow]
    v2 = (w[..., 1:4] ** 2).sum(-1)
    pe = (gam - 1.0) * (w[..., 4] - 0.5 * w[..., 0] * v2)
    r["p_floor"] = int((pe < PRESSURE_FLOOR * prm.pInfCorr).sum())
    if hb.nw > 5:
        r["turb_clip"] = int((w[..., 5] < TURB_CLIP * prm.wInf[5]).sum())
        r["sa_rr_clip"] = int((sa_rr_unclipped(prm, hb) > 10.0).sum())
    return r


def owned_away_from(hb, name, at=None, margin=2):
    """mask of the owned cells more than `margin` cells from the contact discontinuity of a contact regime"""
    d = hb.d
    a = "ijk".index(name[-1])
    c0 = contact_plane(name, (d.nx, d.ny, d.nz)) if at is None else at
    idx = np.arange(2, (d.il, d.jl, d.kl)[a] + 1)
    keep = (idx < c0 - margin) | (idx > c0 - 1 + margin)
    shape = [1, 1, 1]
    shape[a] = -1
    return np.broadcast_to(keep.reshape(shape), (d.nx, d.ny, d.nz))
