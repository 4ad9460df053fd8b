"""Deterministic synthetic structured blocks for parity tests and the benchmark.

The reference's regression meshes are downloaded by ``input_files/get-input-files.sh``
and are not available offline, so the workload is synthetic (SURVEY.md section 8d):

* mesh: analytic curvilinear hexahedral block = Cartesian box + tanh wall-normal
  stretching in k (first cell height ``first_cell`` for RANS) + smooth sinusoidal
  skew of ~10 % of the spacing so that no metric term vanishes; right handed.
  Halo nodes (index 0 and ie) are the analytic continuation of the mapping.
* metrics: face normals by the blockette ``metrics`` formula
  (``src/NKSolver/blockette.F90:881-955``), volumes by ``volume_block``
  (``src/adjoint/adjointExtra.F90:5-177``), both restated in vectorised numpy;
  ``volRef = vol``; ``d2Wall`` = distance of the cell centre to the k=1 plane.
* state: tutorial-wing free stream (M 0.8, alpha 1.8 deg) non-dimensionalised like
  ``referenceState``; smooth 5 % perturbation plus ``default_rng(314)`` noise of 1e-3
  (seed mirrors ``getStatePerturbation(314)``, ``adflow/pyADflow.py:5207``); a
  tanh boundary-layer profile towards the k=1 wall; nuTilde ~ 3 nu_inf away from the
  wall and -> 0 at the wall.
* boundary conditions: NS wall on kMin, symmetry on jMin, far field elsewhere;
  porosities from ``setPorosities`` (``src/preprocessing/preprocessingAPI.F90:567-640``).
"""
import math

import numpy as np

from .layout import HostBlock
from .params import EULER, RANS

BC_SYMM, BC_WALL, BC_FARFIELD, BC_EULERWALL, BC_EXTRAP = 1, 2, 3, 4, 5
IMIN, IMAX, JMIN, JMAX, KMIN, KMAX = 1, 2, 3, 4, 5, 6


def _stretch(zeta, beta):
    return 1.0 + np.tanh(beta * (zeta - 1.0)) / math.tanh(beta)


def _solve_beta(nz_global, first_cell):
    """beta such that the first cell height of the tanh stretching equals first_cell."""
    if first_cell is None:
        return None
    lo, hi = 1e-3, 40.0
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        h = 1.0 + math.tanh(mid * (1.0 / nz_global - 1.0)) / math.tanh(mid)
        if h > first_cell:
            lo = mid
        else:
            hi = mid
    return 0.5 * (lo + hi)


def node_coordinates(nx, ny, nz, origin=(0, 0, 0), global_n=None, first_cell=1e-5, skew=0.1):
    """x(0:ie,0:je,0:ke,3) placed in the uniform box (entries beyond ie unused)."""
    gn = global_n or (nx, ny, nz)
    hb_box = (nx + 4, ny + 4, nz + 4)
    i = np.arange(hb_box[0])[:, None, None]
    j = np.arange(hb_box[1])[None, :, None]
    k = np.arange(hb_box[2])[None, None, :]
    xi = (i - 1 + origin[0]) / gn[0]
    eta = (j - 1 + origin[1]) / gn[1]
    zeta = (k - 1 + origin[2]) / gn[2]
    beta = _solve_beta(gn[2], first_cell)
    zs = zeta if beta is None else _stretch(zeta, beta)
    two_pi = 2.0 * math.pi
    X = xi + (skew / gn[0]) * np.sin(two_pi * eta) * np.cos(1.5 * math.pi * zeta)
    Y = eta + (skew / gn[1]) * np.sin(two_pi * xi + 0.3) * np.cos(math.pi * zeta)
    Z = zs * (1.0 + 0.05 * np.sin(two_pi * xi) * np.sin(two_pi * eta)) + 0.0 * xi * eta
    x = np.zeros(hb_box + (3,), order="F")
    x[..., 0] = X + 0.0 * Y
    x[..., 1] = Y + 0.0 * X
    x[..., 2] = Z
    return x


def compute_metrics(blk):
    """si, sj, sk from x: blockette `metrics`, src/NKSolver/blockette.F90:854-960."""
    d, x = blk.d, blk.x
    fact = 0.5 if blk.right_handed else -0.5

    def cross(v1, v2):
        return fact * np.stack(
            [v1[..., 1] * v2[..., 2] - v1[..., 2] * v2[..., 1],
             v1[..., 2] * v2[..., 0] - v1[..., 0] * v2[..., 2],
             v1[..., 0] * v2[..., 1] - v1[..., 1] * v2[..., 0]], axis=-1)

    I = slice(0, d.ie + 1)
    # i faces: i=0..ie, j=1..je, k=1..ke ; m=j-1, n=k-1
    J, K, M, Nn = slice(1, d.je + 1), slice(1, d.ke + 1), slice(0, d.je), slice(0, d.ke)
    v1 = x[I, J, Nn] - x[I, M, K]
    v2 = x[I, J, K] - x[I, M, Nn]
    blk.si[I, J, K] = cross(v1, v2)
    # j faces: i=1..ie, j=0..je, k=1..ke ; l=i-1, n=k-1
    Ii, L, Jj = slice(1, d.ie + 1), slice(0, d.ie), slice(0, d.je + 1)
    v1 = x[Ii, Jj, Nn] - x[L, Jj, K]
    v2 = x[L, Jj, Nn] - x[Ii, Jj, K]
    blk.sj[Ii, Jj, K] = cross(v1, v2)
    # k faces: i=1..ie, j=1..je, k=0..ke ; l=i-1, m=j-1
    Kk = slice(0, d.ke + 1)
    v1 = x[Ii, J, Kk] - x[L, M, Kk]
    v2 = x[L, J, Kk] - x[Ii, M, Kk]
    blk.sk[Ii, J, Kk] = cross(v1, v2)


def compute_volumes(blk):
    """vol(1:ie,1:je,1:ke): volume_block, src/adjoint/adjointExtra.F90:5-177."""
    d, x = blk.d, blk.x
    Ii, L = slice(1, d.ie + 1), slice(0, d.ie)
    J, M = slice(1, d.je + 1), slice(0, d.je)
    K, Nn = slice(1, d.ke + 1), slice(0, d.ke)
    ijk, imk, imn, ijn = x[Ii, J, K], x[Ii, M, K], x[Ii, M, Nn], x[Ii, J, Nn]
    ljk, lmk, lmn, ljn = x[L, J, K], x[L, M, K], x[L, M, Nn], x[L, J, Nn]
    ctr = 0.125 * (ijk + imk + imn + ijn + ljk + lmk + lmn + ljn)

    def volpym(a, b, c, dd):
        q = ctr - 0.25 * (a + b + c + dd)
        return (q[..., 0] * ((a[..., 1] - c[..., 1]) * (b[..., 2] - dd[..., 2]) - (a[..., 2] - c[..., 2]) * (b[..., 1] - dd[..., 1]))
                + q[..., 1] * ((a[..., 2] - c[..., 2]) * (b[..., 0] - dd[..., 0]) - (a[..., 0] - c[..., 0]) * (b[..., 2] - dd[..., 2]))
                + q[..., 2] * ((a[..., 0] - c[..., 0]) * (b[..., 1] - dd[..., 1]) - (a[..., 1] - c[..., 1]) * (b[..., 0] - dd[..., 0])))

    vp = (volpym(ijk, ijn, imn, imk) + volpym(ljk, lmk, lmn, ljn) + volpym(ijk, ljk, ljn, ijn)
          + volpym(imk, imn, lmn, lmk) + volpym(ijk, imk, lmk, ljk) + volpym(ijn, ljn, lmn, imn))
    blk.vol[...] = 0.0
    blk.vol[Ii, J, K] = np.abs(vp / 6.0)
    # (the haloCellRatio repair of collapsed halo cells never triggers on these meshes)
    blk.volRef[...] = blk.vol


def cell_centres(blk):
    d, x = blk.d, blk.x
    Ii, L = slice(1, d.ie + 1), slice(0, d.ie)
    J, M = slice(1, d.je + 1), slice(0, d.je)
    K, Nn = slice(1, d.ke + 1), slice(0, d.ke)
    c = np.zeros(d.box + (3,), order="F")
    c[Ii, J, K] = 0.125 * (x[Ii, J, K] + x[Ii, M, K] + x[Ii, M, Nn] + x[Ii, J, Nn]
                           + x[L, J, K] + x[L, M, K] + x[L, M, Nn] + x[L, J, Nn])
    # 2nd halo layer: linear extrapolation of the centres (only used to seed the state)
    c[0] = 2 * c[1] - c[2]
    c[d.ib] = 2 * c[d.ie] - c[d.il]
    c[:, 0] = 2 * c[:, 1] - c[:, 2]
    c[:, d.jb] = 2 * c[:, d.je] - c[:, d.jl]
    c[:, :, 0] = 2 * c[:, :, 1] - c[:, :, 2]
    c[:, :, d.kb] = 2 * c[:, :, d.ke] - c[:, :, d.kl]
    return c


def lam_viscosity(prm, p, rho):
    """Sutherland, src/utils/flowUtils.F90:1201-1323."""
    T = p / (prm.RGas * rho)
    return prm.muSuth * ((prm.TSuth + prm.SSuth) / (T + prm.SSuth)) * (T / prm.TSuth) ** 1.5


def eddy_viscosity(prm, w, rlv):
    """saEddyViscosity, src/turbulence/turbUtils.F90:657-712."""
    rnu = w[..., 5] * w[..., 0]
    chi = rnu / rlv
    chi3 = chi**3
    return chi3 / (chi3 + prm.rsaCv1**3) * rnu


def fill_state(blk, prm, seed=314, origin_tag=0, noise=1e-3, amp=0.05, wall_profile=True):
    """Seeded smooth + noisy state in every cell of the box (halos included)."""
    d = blk.d
    c = cell_centres(blk)
    X, Y, Z = c[..., 0], c[..., 1], c[..., 2]
    rng = np.random.default_rng(seed + 7919 * origin_tag)
    nz = lambda: 1.0 + noise * rng.standard_normal(d.box)  # noqa: E731
    two_pi = 2.0 * math.pi
    winf = [prm.wInf[i] for i in range(6)]
    gam = prm.gammaInf
    bl = np.tanh(np.abs(Z) / 0.02) if wall_profile else 1.0
    rho = winf[0] * (1.0 + amp * np.sin(two_pi * X + 1.0) * np.cos(two_pi * Y)) * nz()
    u = winf[1] * (1.0 + amp * np.sin(two_pi * Y + 0.5) * np.cos(math.pi * Z)) * bl * nz()
    v = (winf[2] + amp * winf[1] * np.sin(two_pi * X) * np.sin(two_pi * Z + 0.2)) * bl * nz()
    ww = (winf[3] + amp * winf[1] * np.cos(two_pi * X + 0.7) * np.sin(two_pi * Y)) * bl * nz()
    p = prm.pInf * (1.0 + amp * np.cos(two_pi * X) * np.cos(two_pi * Y + 0.4) * np.cos(math.pi * Z)) * nz()
    blk.w[..., 0], blk.w[..., 1], blk.w[..., 2], blk.w[..., 3] = rho, u, v, ww
    blk.p[...] = p
    blk.w[..., 4] = p / (gam - 1.0) + 0.5 * rho * (u * u + v * v + ww * ww)
    if blk.nw > 5:
        nu_inf = prm._muInf / prm.rhoInf
        g = np.tanh(np.abs(Z) / 0.01) if wall_profile else 1.0
        blk.w[..., 5] = 3.0 * nu_inf * (g + 1e-3) * nz()
    if prm.equations != EULER:
        blk.rlv[...] = lam_viscosity(prm, blk.p, blk.w[..., 0])
    if prm.equations == RANS:
        blk.rev[...] = eddy_viscosity(prm, blk.w, blk.rlv)


def make_block(nx, ny, nz, prm, origin=(0, 0, 0), global_n=None, first_cell="auto", seed=314,
               origin_tag=0, physical_faces=(IMIN, IMAX, JMIN, JMAX, KMIN, KMAX)):
    """One synthetic block: geometry + BC description + seeded state."""
    nw = 6 if prm.equations == RANS else 5
    blk = HostBlock(nx, ny, nz, nw=nw)
    if first_cell == "auto":
        first_cell = 1e-5 if prm.equations == RANS else None
    blk.x[...] = node_coordinates(nx, ny, nz, origin, global_n, first_cell)
    compute_metrics(blk)
    compute_volumes(blk)
    d = blk.d
    cc = cell_centres(blk)
    blk.d2Wall[...] = 1.0
    blk.d2Wall[d.owned()] = np.abs(cc[d.owned() + (2,)])
    # subfaces: wall on kMin, symmetry on jMin, far field elsewhere (SURVEY 8d)
    blk.subfaces = []
    # physical_faces: the faces that carry a physical BC (default layout), or a dict face -> bcType
    for face in physical_faces:
        if isinstance(physical_faces, dict):
            bc = physical_faces[face]
            if prm.equations == EULER and bc in (BC_WALL, 6):
                bc = BC_EULERWALL
        else:
            bc = BC_FARFIELD
            if face == KMIN:
                bc = BC_WALL if prm.equations != EULER else BC_EULERWALL
            elif face == JMIN:
                bc = BC_SYMM
        blk.subfaces.append(make_subface(blk, face, bc, prm))
        if bc in (BC_WALL, BC_EULERWALL, BC_EXTRAP, 6):  # setPorosities
            if face == IMIN: blk.porI[1, :, :] = 0
            if face == IMAX: blk.porI[d.il, :, :] = 0
            if face == JMIN: blk.porJ[:, 1, :] = 0
            if face == JMAX: blk.porJ[:, d.jl, :] = 0
            if face == KMIN: blk.porK[:, :, 1] = 0
            if face == KMAX: blk.porK[:, :, d.kl] = 0
    fill_state(blk, prm, seed=seed, origin_tag=origin_tag)
    return blk


def make_subface(blk, face, bc, prm=None, iblank=None):
    """BCData of one whole block face: cell range 1:ie x 1:je of the two in-plane
    directions (halo-extended like icBeg:icEnd, src/utils/utils.F90:895-900) and the
    unit outward normal from the face's s-vector (boundaryNormals,
    src/adjoint/adjointExtra.F90).  iblank: the surface blanking BCData%iblank over that
    range (key "iblank"); absent means 1 everywhere."""
    d = blk.d
    if face in (IMIN, IMAX):
        n1, n2 = d.je, d.ke
        s = blk.si[1 if face == IMIN else d.il, :, :, :]
    elif face in (JMIN, JMAX):
        n1, n2 = d.ie, d.ke
        s = blk.sj[:, 1 if face == JMIN else d.jl, :, :]
    else:
        n1, n2 = d.ie, d.je
        s = blk.sk[:, :, 1 if face == KMIN else d.kl, :]
    s = s[1:n1 + 1, 1:n2 + 1, :]
    mult = -1.0 if face in (IMIN, JMIN, KMIN) else 1.0
    mag = np.sqrt((s * s).sum(axis=-1))
    mag = np.where(mag > 0, mag, 1.0)
    norm = np.asfortranarray(mult * s / mag[..., None])
    sub = {"bcType": bc, "faceId": face, "icBeg": 1, "icEnd": n1, "jcBeg": 1, "jcEnd": n2, "norm": norm}
    if iblank is not None:
        assert np.shape(iblank) == (n1, n2), np.shape(iblank)
        sub["iblank"] = np.asfortranarray(iblank, dtype=np.int32)
    a, c = np.meshgrid(np.arange(n1), np.arange(n2), indexing="ij")
    wig = np.sin(0.37 * a) * np.cos(0.23 * c)          # smooth in-plane variation of the prescribed data
    if bc == 6:  # isothermal wall: BCData%TNS_Wall, non-dimensional (T_inf = 1), smooth 5 % variation
        sub["TNSWall"] = np.asfortranarray(1.08 + 0.05 * wig)
    if prm is not None and bc in (7, 8, 9, 10):
        F = np.asfortranarray
        g, R = prm.gammaInf, prm.RGas
        rho, u, v, w_ = prm.wInf[0], prm.wInf[1], prm.wInf[2], prm.wInf[3]
        if bc == 7:      # subsonic outflow: static pressure
            sub["ps"] = F(prm.pInf * (0.97 + 0.02 * wig))
        if bc == 9:      # supersonic inflow: full state
            sub.update(rho=F(rho * (1.02 + 0.01 * wig)), velx=F(u * (1.5 + 0.02 * wig)), vely=F(v + 0.01 * wig),
                       velz=F(w_ + 0.02 * wig), ps=F(prm.pInf * (1.05 + 0.01 * wig)))
        if bc == 8:      # subsonic inflow; treatment chosen by the face parity so that both branches are exercised
            sub["subsonicInletTreatment"] = 1 if face % 2 == 1 else 2
            m2 = (u * u + v * v + w_ * w_) / (g * prm.pInf / rho)
            tt = (prm.pInf / (R * rho)) * (1.0 + 0.5 * (g - 1.0) * m2)
            pt = prm.pInf * (1.0 + 0.5 * (g - 1.0) * m2) ** (g / (g - 1.0))
            dirn = -norm + 0.05 * wig[..., None]
            dirn = dirn / np.sqrt((dirn * dirn).sum(-1))[..., None]
            sub.update(ptInlet=F(pt * (1.0 + 0.01 * wig)), ttInlet=F(tt * (1.0 + 0.005 * wig)),
                       htInlet=F(g / (g - 1.0) * R * tt * (1.0 + 0.005 * wig)), flowXdirInlet=F(dirn[..., 0]),
                       flowYdirInlet=F(dirn[..., 1]), flowZdirInlet=F(dirn[..., 2]),
                       rho=F(rho * (1.01 + 0.01 * wig)), velx=F(-0.3 * norm[..., 0] + 0.01 * wig),
                       vely=F(-0.3 * norm[..., 1]), velz=F(-0.3 * norm[..., 2]))
        if bc in (8, 9) and prm.equations == RANS:
            sub["turbInlet"] = F(prm.wInf[5] * (1.0 + 0.1 * wig))
    return sub


# ---------------------------------------------------------------------------------------------
# multigrid: coarse block of a synthetic block (what createCoarseBlocks, src/preprocessing/coarseUtils.F90, sets up)
def mg_kept_nodes(n_cells):
    """iCo(1:il): fine nodes kept on the coarse level.  Every other node; the last node is always kept, so an odd
    number of cells ends in an irregular coarse cell made of ONE fine cell (weight 1/2, coarseUtils.F90:283-296)."""
    il = n_cells + 1
    keep = np.zeros(il + 1, dtype=bool)      # index 1..il
    keep[1:il + 1:2] = True
    keep[il] = True
    return keep


def mg_tables_1d(keep, ie_c, ie_f, ib_f):
    """mgIFine(1:ie_c, 2), mgIWeight(2:il_c), mgICoarse(2:il_f, 2) of one direction from iCo = `keep`
    (coarseUtils.F90:270-352); Fortran index == numpy index."""
    il_f = keep.size - 1
    fine = np.zeros((ie_c + 1, 2), dtype=np.int32)
    wgt = np.zeros(ie_c + 1)
    coarse = np.zeros((ie_f + 1, 2), dtype=np.int32)
    fine[1] = (0, 1)
    fine[ie_c] = (ie_f, ib_f)
    ii = 2
    for i in range(2, il_f + 1):
        if keep[i]:
            if keep[i - 1]:
                fine[ii] = (i, i); wgt[ii] = 0.5
            else:
                fine[ii] = (i - 1, i); wgt[ii] = 1.0
            ii += 1
    ii = 2
    for i in range(2, il_f + 1):
        if keep[i]:
            coarse[i] = (ii, ii) if keep[i - 1] else (ii, ii + 1)
            ii += 1
        else:
            coarse[i] = (ii, ii - 1)
    return fine, wgt, coarse


def make_coarse_block(fine, prm, keeps=None):
    """The next coarser level of `fine`: nodes = the kept fine nodes (halo nodes extrapolated), metrics, volumes,
    wall distance (volume average), porosities and boundary subfaces of the same types, restriction tables on the
    coarse block and interpolation tables on `fine` (fine.mg is updated).  The state is left zero: it is the
    output of the restriction.  keeps: iCo, jCo, kCo (as mg_kept_nodes returns them); default mg_kept_nodes."""
    df = fine.d
    if keeps is None:
        keeps = [mg_kept_nodes(n) for n in (df.nx, df.ny, df.nz)]
    nc = [int(k.sum()) - 1 for k in keeps]
    blk = HostBlock(*nc, nw=fine.nw, right_handed=fine.right_handed)
    blk.level = fine.level + 1
    d = blk.d
    idx = [np.flatnonzero(k) for k in keeps]                      # fine node index of coarse node 1..il_c
    x = np.zeros(d.box + (3,), order="F")
    x[1:d.il + 1, 1:d.jl + 1, 1:d.kl + 1] = fine.x[np.ix_(idx[0], idx[1], idx[2])]
    x[0], x[d.ie] = 2 * x[1] - x[2], 2 * x[d.il] - x[d.il - 1]
    x[:, 0], x[:, d.je] = 2 * x[:, 1] - x[:, 2], 2 * x[:, d.jl] - x[:, d.jl - 1]
    x[:, :, 0], x[:, :, d.ke] = 2 * x[:, :, 1] - x[:, :, 2], 2 * x[:, :, d.kl] - x[:, :, d.kl - 1]
    blk.x[...] = x
    compute_metrics(blk)
    compute_volumes(blk)
    tabs = [mg_tables_1d(keeps[a], (d.ie, d.je, d.ke)[a], (df.ie, df.je, df.ke)[a], (df.ib, df.jb, df.kb)[a]) for a in range(3)]
    for a, nm in enumerate("IJK"):
        blk.mg["mg%sFine" % nm], blk.mg["mg%sWeight" % nm] = tabs[a][0], tabs[a][1]
        fine.mg["mg%sCoarse" % nm] = tabs[a][2]
    # wall distance of the coarse cells: volume-weighted average of the fine cells
    ow = d.owned()
    fI, fJ, fK = (blk.mg["mg%sFine" % nm] for nm in "IJK")
    num = np.zeros((d.nx, d.ny, d.nz)); den = np.zeros_like(num)
    for a in (0, 1):
        for b_ in (0, 1):
            for c in (0, 1):
                sel = np.ix_(fI[2:d.il + 1, a], fJ[2:d.jl + 1, b_], fK[2:d.kl + 1, c])
                num += fine.vol[sel] * fine.d2Wall[sel]; den += fine.vol[sel]
    blk.d2Wall[...] = 1.0
    blk.d2Wall[ow] = num / den
    blk.subfaces = []
    for s in fine.subfaces:
        face, bc = s["faceId"], s["bcType"]
        blk.subfaces.append(make_subface(blk, face, bc, prm))
        if bc in (BC_WALL, BC_EULERWALL, BC_EXTRAP, 6):
            if face == IMIN: blk.porI[1, :, :] = 0
            if face == IMAX: blk.porI[d.il, :, :] = 0
            if face == JMIN: blk.porJ[:, 1, :] = 0
            if face == JMAX: blk.porJ[:, d.jl, :] = 0
            if face == KMIN: blk.porK[:, :, 1] = 0
            if face == KMAX: blk.porK[:, :, d.kl] = 0
    # a benign state so that halo cells never hold zeros (divisions): free stream, overwritten by the restriction
    for l in range(fine.nw):
        blk.w[..., l] = prm.wInf[l]
    blk.w[..., 4] = prm.wInf[4]
    blk.p[...] = prm.pInf
    blk.rlv[...] = lam_viscosity(prm, blk.p, blk.w[..., 0]) if prm.equations != EULER else 0.0
    if prm.equations == RANS:
        blk.rev[...] = eddy_viscosity(prm, blk.w, blk.rlv)
    return blk
