"""Test meshes of the topologies real ADflow meshes have and the synthetic box has not.

* ``o_grid``: an annulus about a cylinder round the x axis.  i is axial, j runs once round the axis and closes on
  itself (a periodic 1-to-1 cut from jMax back to jMin of the same block), k is radial with the wall on kMin.
* ``polar_grid``: the same layout with r starting at 0, so kMin is collapsed onto the axis (a polar singular line,
  ``sk`` exactly 0, wedge cells next to it) and carries the polar symmetry BC; the wall is the iMin disc.
* ``permute_axes``: a block as its cyclic axis permutation, so that the same physical problem has its wall normal along
  i or j instead of k.
* ``self_periodic_pattern``: the donor / halo lists of the periodic cut in the list format of ``adflow_b200.halo``.

Nodes are placed like the reference's preprocessing places them (``xhalo``, src/preprocessing/preprocessingAPI.F90:
1042-1299): owned nodes from the mapping, halo nodes extrapolated linearly, then mirrored about the plane of each
symmetry face whose corner diagonals span one, then copied from across the cut (``exchangeCoor``).  The polar BC is not
a symmetry plane there, so its halo nodes are the extrapolation, which mirrors them through the axis; on an i face of
the O-grid node jl is node 1, the corner diagonals are parallel, and xhalo leaves the extrapolation too.  So a halo
cell across the cut has its donor's geometry bit for bit, and the state handed out has been through the cut's exchange
once.
"""
import math

import numpy as np

from adflow_b200 import synthetic as syn
from adflow_b200.halo import exchange_numpy
from adflow_b200.layout import HostBlock
from adflow_b200.params import EULER, RANS

BC_SYMMPOLAR = 11
WALL_TYPES = (syn.BC_WALL, syn.BC_EULERWALL, syn.BC_EXTRAP, 6)   # the BCs setPorosities closes the face for


def _xhalo(x, d, cut_axis=None, symm_faces=()):
    """halo nodes of xhalo: linear extrapolation in i, then j (with the i halos), then k (with both); then the halo
    nodes of the symmetry faces `symm_faces` (whole faces) mirrored about the plane through the face's corner diagonals;
    then, along `cut_axis`, the halo nodes copied from across the periodic cut (exchangeCoor; node l == node 1 already)"""
    ends = ((d.ie, d.il, d.nx), (d.je, d.jl, d.ny), (d.ke, d.kl, d.nz))
    full = [slice(0, d.ie + 1), slice(0, d.je + 1), slice(0, d.ke + 1)]

    def at(sl, a, idx):
        s = list(sl)
        s[a] = idx
        return tuple(s)

    for a in range(3):
        e, l_, n = ends[a]
        sl = [full[b] if b < a else slice(1, ends[b][1] + 1) for b in range(3)]   # later directions: owned nodes only
        x[at(sl, a, 0)] = 2.0 * x[at(sl, a, 1)] - x[at(sl, a, 2)]
        x[at(sl, a, e)] = 2.0 * x[at(sl, a, l_)] - x[at(sl, a, n)]
    for face in symm_faces:
        a, high = (face - 1) // 2, (face - 1) % 2
        e, l_, n = ends[a]
        x0, x1, x2 = (x[at(full, a, q)] for q in ((e, l_, n) if high else (0, 1, 2)))
        (p, q) = [ends[b][1] for b in range(3) if b != a]
        v1, v2 = x1[p, q] - x1[1, 1], x1[p, 1] - x1[1, q]
        norm = np.cross(v1, v2)
        length = math.sqrt((norm * norm).sum())
        if length > 1e-25:          # eps: a singular face (corner diagonals parallel) keeps the extrapolation
            norm = norm / length
            dot = 2.0 * ((x1 - x2) * norm).sum(-1)
            x0[...] = x2 + dot[..., None] * norm
    if cut_axis is not None:
        e, l_, n = ends[cut_axis]
        x[at(full, cut_axis, 0)] = x[at(full, cut_axis, n)]
        x[at(full, cut_axis, e)] = x[at(full, cut_axis, 2)]


def _cell_average(blk, nodal):
    """a nodal scalar (0:ie, 0:je, 0:ke) averaged to the cells 1:ie like the cell centres, second halos
    extrapolated linearly (synthetic.cell_centres)"""
    d = blk.d
    Ii, L = slice(1, d.ie + 1), slice(0, d.ie)
    J, M = slice(1, d.je + 1), slice(0, d.je)
    K, Nn = slice(1, d.ke + 1), slice(0, d.ke)
    c = np.zeros(d.box, order="F")
    c[Ii, J, K] = 0.125 * (nodal[Ii, J, K] + nodal[Ii, M, K] + nodal[Ii, M, Nn] + nodal[Ii, J, Nn]
                           + nodal[L, J, K] + nodal[L, M, K] + nodal[L, M, Nn] + nodal[L, J, Nn])
    c[0] = 2 * c[1] - c[2]
    c[d.ib] = 2 * c[d.ie] - c[d.il]
    c[:, 0] = 2 * c[:, 1] - c[:, 2]
    c[:, d.jb] = 2 * c[:, d.je] - c[:, d.jl]
    c[:, :, 0] = 2 * c[:, :, 1] - c[:, :, 2]
    c[:, :, d.kb] = 2 * c[:, :, d.ke] - c[:, :, d.kl]
    return c


def _radii(n, r0, r1, first_cell):
    """n + 1 node radii from r0 to r1, tanh-stretched towards r0 to a first cell of first_cell (None: uniform)"""
    zeta = np.arange(n + 1) / n
    beta = syn._solve_beta(n, None if first_cell is None else first_cell / (r1 - r0))
    s = zeta if beta is None else syn._stretch(zeta, beta)
    return r0 + (r1 - r0) * s


def _revolved_block(nx, ny, nz, prm, axial, radial, wobble, symm_faces=()):
    """block of nodes x = axial[i], (y, z) = r (cos t, -sin t) with t = 2 pi (j-1) / ny and r = radial[k] * (1 +
    wobble * s(k) sin(2 pi x) cos t), s rising from 0 on the first radial node; right handed (i, j, k) =
    (axial, circumferential, radial)"""
    nw = 6 if prm.equations == RANS else 5
    blk = HostBlock(nx, ny, nz, nw=nw)
    d = blk.d
    X = np.asarray(axial)[:, None, None]
    t = 2.0 * math.pi * np.arange(ny)[None, :, None] / ny
    r = np.asarray(radial)[None, None, :]
    s = (r - r[..., :1]) / (r[..., -1:] - r[..., :1])
    rr = r * (1.0 + wobble * s * np.sin(2.0 * math.pi * X) * np.cos(t))
    x = np.zeros(d.box + (3,), order="F")
    own = (slice(1, d.il + 1), slice(1, d.jl), slice(1, d.kl + 1))
    x[own + (0,)] = X + 0.0 * t * r
    x[own + (1,)] = rr * np.cos(t)
    x[own + (2,)] = -rr * np.sin(t)
    x[:, d.jl] = x[:, 1]                      # the cut: node jl is node 1
    _xhalo(x, d, cut_axis=1, symm_faces=symm_faces)
    blk.x[...] = x
    syn.compute_metrics(blk)
    syn.compute_volumes(blk)
    return blk


def _subfaces(blk, prm, faces):
    blk.subfaces = []
    d = blk.d
    for face, bc in faces.items():
        if prm.equations == EULER and bc in (syn.BC_WALL, 6):
            bc = syn.BC_EULERWALL
        blk.subfaces.append(syn.make_subface(blk, face, bc, prm))
        if bc in WALL_TYPES:                  # setPorosities
            if face == syn.IMIN: blk.porI[1, :, :] = 0
            if face == syn.IMAX: blk.porI[d.il, :, :] = 0
            if face == syn.KMIN: blk.porK[:, :, 1] = 0
            if face == syn.KMAX: blk.porK[:, :, d.kl] = 0
    blk.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (syn.BC_WALL, 6) else 1)   # viscous subfaces first


def _seed_state(blk, prm, seed, wall_dist):
    """synthetic.fill_state without its z = 0 wall profile, then a boundary-layer profile in the wall distance of
    every cell (halos included) and one pass of the periodic cut's exchange"""
    syn.fill_state(blk, prm, seed=seed, wall_profile=False)
    bl = np.tanh(np.abs(wall_dist) / 0.02)
    blk.w[..., 1:4] *= bl[..., None]
    rho, u, v, w_ = blk.w[..., 0], blk.w[..., 1], blk.w[..., 2], blk.w[..., 3]
    blk.w[..., 4] = blk.p / (prm.gammaInf - 1.0) + 0.5 * rho * (u * u + v * v + w_ * w_)
    if blk.nw > 5:
        blk.w[..., 5] *= (np.tanh(np.abs(wall_dist) / 0.01) + 1e-3) / (1.0 + 1e-3)
        blk.rev[...] = syn.eddy_viscosity(prm, blk.w, blk.rlv)
    exchange_numpy([blk], self_periodic_pattern(blk, 2), lambda hb: state_vars(hb))


def state_vars(hb):
    """every cell array the state consists of: w, p, rlv, rev"""
    return [hb.w[..., l] for l in range(hb.nw)] + [hb.p, hb.rlv, hb.rev]


def o_grid(nx, ny, nz, prm, r_in=0.5, r_out=1.5, length=1.0, first_cell="auto", i_faces=(syn.BC_SYMM, syn.BC_FARFIELD),
           wobble=0.05, seed=314):
    """annulus r_in..r_out about the x axis, 0 <= x <= length; wall on kMin (the cylinder), far field on kMax,
    i_faces on iMin / iMax, the j faces joined to each other.  first_cell: radial height of the wall cells
    ("auto": 1e-5 for RANS, uniform otherwise).  d2Wall: radial distance of the cell from the cylinder."""
    if first_cell == "auto":
        first_cell = 1e-5 if prm.equations == RANS else None
    rad = _radii(nz, r_in, r_out, first_cell)
    symm = [f for f, bc in zip((syn.IMIN, syn.IMAX), i_faces) if bc == syn.BC_SYMM]
    blk = _revolved_block(nx, ny, nz, prm, length * np.arange(nx + 1) / nx, rad, wobble, symm)
    d = blk.d
    dist = np.zeros((d.ie + 1, d.je + 1, d.ke + 1))
    dist[:, :, 1:d.kl + 1] = (rad - r_in)[None, None, :]
    dist[:, :, 0] = 2 * dist[:, :, 1] - dist[:, :, 2]
    dist[:, :, d.ke] = 2 * dist[:, :, d.kl] - dist[:, :, d.nz]
    cd = _cell_average(blk, dist)
    blk.d2Wall[...] = 1.0
    blk.d2Wall[d.owned()] = cd[d.owned()]
    _subfaces(blk, prm, {syn.IMIN: i_faces[0], syn.IMAX: i_faces[1], syn.KMIN: syn.BC_WALL, syn.KMAX: syn.BC_FARFIELD})
    _seed_state(blk, prm, seed, cd)
    return blk


def polar_grid(nx, ny, nz, prm, radius=1.0, length=1.0, first_cell="auto", wobble=0.05, seed=314):
    """cylinder 0 <= r <= radius, 0 <= x <= length: kMin collapsed onto the axis with the polar symmetry BC, wall on
    the iMin disc (axial first cell of first_cell, "auto" as in o_grid), far field on iMax and kMax, the j faces
    joined to each other.  d2Wall: axial distance of the cell from the disc."""
    if first_cell == "auto":
        first_cell = 1e-5 if prm.equations == RANS else None
    axial = _radii(nx, 0.0, length, first_cell)
    blk = _revolved_block(nx, ny, nz, prm, axial, _radii(nz, 0.0, radius, None), wobble)
    d = blk.d
    cd = _cell_average(blk, blk.x[..., 0][:d.ie + 1, :d.je + 1, :d.ke + 1])
    blk.d2Wall[...] = 1.0
    blk.d2Wall[d.owned()] = cd[d.owned()]
    _subfaces(blk, prm, {syn.IMIN: syn.BC_WALL, syn.IMAX: syn.BC_FARFIELD, syn.KMIN: BC_SYMMPOLAR, syn.KMAX: syn.BC_FARFIELD})
    _seed_state(blk, prm, seed, cd)
    return blk


def coarse_level(fine, prm, cut_axis=1):
    """synthetic.make_coarse_block of a block with a periodic cut: the kept nodes keep node l == node 1, and the halo
    nodes across the cut are copied from the other side instead of extrapolated (geometry and BCData again)"""
    blk = syn.make_coarse_block(fine, prm)
    d = blk.d
    x = blk.x.copy()
    _xhalo(x, d, cut_axis, [s["faceId"] for s in fine.subfaces if s["bcType"] == syn.BC_SYMM])
    blk.x[...] = x
    syn.compute_metrics(blk)
    syn.compute_volumes(blk)
    blk.subfaces = [dict(syn.make_subface(blk, s["faceId"], s["bcType"], prm)) for s in fine.subfaces]
    return blk


def self_periodic_pattern(hb, layers=2, axis=1):
    """donor / halo lists of a block whose two faces normal to `axis` are one periodic cut (node l == node 1).
    layers 2 (the finest level, commPatternCell_2nd): both halo layers across the cut over the whole box of the
    other two directions, so the edge and corner halos along the cut come with them; layers 1 (coarse levels,
    commPatternCell_1st): the first halos, over 1:ie of the other directions.  Entries i fastest, then j, k."""
    d = hb.d
    n, e, b = (d.nx, d.ny, d.nz)[axis], (d.ie, d.je, d.ke)[axis], (d.ib, d.jb, d.kb)[axis]
    pairs = [(1, n + 1), (e, 2)] + ([(0, n), (b, 3)] if layers == 2 else [])
    lo, hi = (0, np.array([d.ib, d.jb, d.kb])) if layers == 2 else (1, np.array([d.ie, d.je, d.ke]))
    halo, donor = [], []
    rng = [np.arange(lo, hi[a] + 1) for a in range(3)]
    for h, dn in pairs:
        rng[axis] = np.array([h])
        kk, jj, ii = np.meshgrid(rng[2], rng[1], rng[0], indexing="ij")
        idx = np.stack([ii.ravel(), jj.ravel(), kk.ravel()], axis=1)
        src = idx.copy()
        src[:, axis] = dn
        halo.append(idx); donor.append(src)
    halo, donor = np.concatenate(halo), np.concatenate(donor)
    order = np.lexsort((halo[:, 0], halo[:, 1], halo[:, 2]))
    as4 = lambda a: np.ascontiguousarray(np.column_stack([np.zeros(len(a)), a]), dtype=np.int32)  # noqa: E731
    z = np.zeros(0, dtype=np.int32)
    return {"nbrRank": z, "sendCount": z, "recvCount": z, "sendList": np.zeros((0, 4), np.int32),
            "recvList": np.zeros((0, 4), np.int32), "donorList": as4(donor[order]), "haloList": as4(halo[order])}


# ---------------------------------------------------------------------------------------------------------------------
# cyclic axis permutations
CYCLIC = ((0, 1, 2), (1, 2, 0), (2, 0, 1))
_AXIS_NAMED = (("si", "sj", "sk"), ("radI", "radJ", "radK"), ("porI", "porJ", "porK"))


def inverse(perm):
    inv = [0, 0, 0]
    for q, a in enumerate(perm):
        inv[a] = q
    return tuple(inv)


def permute_box(a, perm):
    """a box array with new axis q = old axis perm[q] (trailing components kept)"""
    return np.asfortranarray(np.transpose(a, tuple(perm) + tuple(range(3, a.ndim))))


def permute_axes(hb, perm):
    """hb as the block whose direction q is hb's direction perm[q]: every array, the arrays named after a
    direction (si/sj/sk, radI/J/K, porI/J/K, the per-direction components of dss and wallTau), the subfaces (face
    ids, in-plane ranges, BCData arrays in the in-plane index order of the new face) and the multigrid tables.
    Only cyclic permutations: they keep a right-handed block right handed."""
    perm = tuple(perm)
    assert perm in CYCLIC, perm
    n = (hb.d.nx, hb.d.ny, hb.d.nz)
    out = HostBlock(*(n[a] for a in perm), nw=hb.nw, right_handed=hb.right_handed)
    out.level = hb.level
    for name in ["w", "dw", "iblank"] + HostBlock.REAL + HostBlock.VEC + ["porI", "porJ", "porK"]:
        setattr(out, name, permute_box(getattr(hb, name), perm))
    for names in _AXIS_NAMED:
        for q in range(3):
            setattr(out, names[q], permute_box(getattr(hb, names[perm[q]]), perm))
    out.dss = np.asfortranarray(out.dss[..., list(perm)])
    out.wallTau = np.asfortranarray(np.concatenate([out.wallTau[..., 9 * a:9 * a + 9] for a in perm], axis=-1))
    inv = inverse(perm)
    out.subfaces = []
    for s in hb.subfaces:
        a, side = (s["faceId"] - 1) // 2, (s["faceId"] - 1) % 2
        b1, b2 = [b for b in range(3) if b != a]
        s2 = dict(s, faceId=2 * inv[a] + 1 + side)
        if inv[b1] > inv[b2]:                 # the new face's first in-plane direction is the old second one
            s2["icBeg"], s2["icEnd"], s2["jcBeg"], s2["jcEnd"] = s["jcBeg"], s["jcEnd"], s["icBeg"], s["icEnd"]
            for k, v in s.items():
                if isinstance(v, np.ndarray):
                    s2[k] = np.asfortranarray(np.swapaxes(v, 0, 1))
        out.subfaces.append(s2)
    for nm in ("Fine", "Weight", "Coarse"):
        for q in range(3):
            key = "mg%s%s" % ("IJK"[perm[q]], nm)
            if key in hb.mg:
                out.mg["mg%s%s" % ("IJK"[q], nm)] = hb.mg[key].copy()
    return out


def unpermute(a, perm):
    """a box array of permute_axes(hb, perm) back in hb's index order"""
    return permute_box(a, inverse(perm))
