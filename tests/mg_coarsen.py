"""The reference's coarsening of one block (createCoarseBlocks, src/preprocessing/coarseUtils.F90), for the tests.

synthetic.make_coarse_block keeps every other node from the left plus the last one on every level, and gives every
coarse face one whole subface.  The reference instead
* keeps both block ends and the end nodes inBeg/inEnd, jnBeg/jnEnd, knBeg/knEnd of every subface of the finer level
  (:114-129), so a face split into pieces stays split;
* fills in every other node from the left or from the right, alternating from one level to the next (iCoarsened,
  :131-193); a direction whose coarsening halves the cell count counts as regular again (:237-246), and the next level
  starts from the left;
* maps every subface's node range through imap (:404-490); the cell ranges follow as in utils.F90:895-900, extended
  into the halos at block edges only.
So an irregular coarse cell (one fine cell, restriction weight 1/2) can sit inside a line, next to a subface end, or at
the min end of a right-started level, where the prolongation of its fine cells reads the coarse halo."""
import numpy as np

from adflow_b200 import synthetic as syn

REGULAR, LEFT, RIGHT = 0, -1, 1
BOUND_FLUX_BCS = (syn.BC_WALL, syn.BC_EULERWALL, syn.BC_EXTRAP, 6)
# the block directions of the two in-plane ranges (icBeg:icEnd, jcBeg:jcEnd) of a subface, per face id
IN_PLANE = {1: (1, 2), 2: (1, 2), 3: (0, 2), 4: (0, 2), 5: (0, 1), 6: (0, 1)}


def node_ranges(hb, s):
    """[(nBeg, nEnd)] of subface s in the three block directions (inBeg:inEnd, jnBeg:jnEnd, knBeg:knEnd)"""
    d = hb.d
    ls = (d.il, d.jl, d.kl)
    axis = (s["faceId"] - 1) // 2
    n = ls[axis] if s["faceId"] % 2 == 0 else 1
    out = [(n, n)] * 3
    for (a, (beg, end)) in zip(IN_PLANE[s["faceId"]], ((s["icBeg"], s["icEnd"]), (s["jcBeg"], s["jcEnd"]))):
        out[a] = (max(beg, 2) - 1, min(end, ls[a]))
    return out


def kept_nodes(n_cells, ends, finer):
    """iCo(1:il) of one direction and the coarsening of the coarse level: `ends` are the subface end nodes of the finer
    level, `finer` its coarsening (REGULAR, LEFT or RIGHT)"""
    il = n_cells + 1
    keep = np.zeros(il + 1, dtype=bool)       # index 1..il
    keep[1] = keep[il] = True
    keep[list(ends)] = True
    if finer == LEFT:
        started = RIGHT
        for i in range(il - 1, 1, -1):
            if not keep[i + 1]:
                keep[i] = True
    else:
        started = LEFT
        for i in range(2, il):
            if not keep[i - 1]:
                keep[i] = True
    if n_cells == 2 * (int(keep.sum()) - 1):
        started = REGULAR
    return keep, started


def coarse_block(fine, prm, coarsened=(REGULAR,) * 3):
    """The next coarser level of `fine` as the reference builds it; `coarsened`: how each direction of `fine` itself
    was coarsened (REGULAR for the finest level).  Returns the coarse HostBlock and its coarsening per direction."""
    d = fine.d
    ranges = [node_ranges(fine, s) for s in fine.subfaces]
    keeps, started = [], []
    for a, n in enumerate((d.nx, d.ny, d.nz)):
        ends = {e for r in ranges for e in r[a]}
        k, st = kept_nodes(n, ends, coarsened[a])
        keeps.append(k)
        started.append(st)
    blk = syn.make_coarse_block(fine, prm, keeps=keeps)
    dc = blk.d
    imap = [np.cumsum(k) for k in keeps]      # imap(i) for a kept node i
    lc, ec = (dc.il, dc.jl, dc.kl), (dc.ie, dc.je, dc.ke)
    blk.porI[1], blk.porI[dc.il] = 1, 1
    blk.porJ[:, 1], blk.porJ[:, dc.jl] = 1, 1
    blk.porK[:, :, 1], blk.porK[:, :, dc.kl] = 1, 1
    subs = []
    for s, r in zip(fine.subfaces, ranges):
        face, bc = s["faceId"], s["bcType"]
        cr = {}
        for a in range(3):
            nb, ne = int(imap[a][r[a][0]]), int(imap[a][r[a][1]])
            cr[a] = (1 if nb == 1 else nb + 1, ec[a] if ne == lc[a] else ne)
        (a0, a1) = IN_PLANE[face]
        sub = syn.make_subface(blk, face, bc, prm)
        (b0, e0), (b1, e1) = cr[a0], cr[a1]
        for key, v in sub.items():
            if isinstance(v, np.ndarray):
                sub[key] = np.asfortranarray(v[b0 - 1:e0, b1 - 1:e1])
        sub.update(icBeg=b0, icEnd=e0, jcBeg=b1, jcEnd=e1)
        subs.append(sub)
        if bc in BOUND_FLUX_BCS:              # setPorosities over the owned faces of the subface
            axis = (face - 1) // 2
            sl = [slice(max(cr[a][0], 2), min(cr[a][1], lc[a]) + 1) for a in range(3)]
            sl[axis] = lc[axis] if face % 2 == 0 else 1
            (blk.porI, blk.porJ, blk.porK)[axis][tuple(sl)] = 0
    blk.subfaces = sorted(subs, key=lambda s_: 0 if s_["bcType"] in (syn.BC_WALL, 6) else 1)
    return blk, tuple(started)


def coarse_levels(fine, prm, nlev):
    """[fine, level 2, ..., level nlev] coarsened as the reference does, and the coarsening of every level"""
    levels, coarsened = [fine], [(REGULAR,) * 3]
    for _ in range(nlev - 1):
        blk, st = coarse_block(levels[-1], prm, coarsened[-1])
        levels.append(blk)
        coarsened.append(st)
    return levels, coarsened


_SYMM, _WALL, _FAR, _EXTRAP, _ISOWALL, _SUBOUT, _SUBIN, _SUPIN, _SUPOUT = 1, 2, 3, 5, 6, 7, 8, 9, 10
# inout: subsonic inflow with total conditions (the odd face iMin), subsonic and supersonic outflow, symmetry, wall, far
# field.  supin: supersonic inflow, extrapolation, isothermal wall, subsonic inflow with mass flow (the even face jMax).
INOUT = {syn.IMIN: _SUBIN, syn.IMAX: _SUBOUT, syn.JMIN: _SYMM, syn.JMAX: _SUPOUT, syn.KMIN: _WALL, syn.KMAX: _FAR}
SUPIN = {syn.IMIN: _SUPIN, syn.IMAX: _EXTRAP, syn.JMIN: _ISOWALL, syn.JMAX: _SUBIN, syn.KMIN: _FAR, syn.KMAX: _SYMM}


def layout_levels(layout, shape, options=None, nlev=2, fields=None, seed=314):
    """parameters and the levels [fine, 2, ...] of a block with boundary layout `layout`: "inout", "supin", "mixed",
    "many" (util.MIXED / MANY on the default layout), "polar" (meshes.polar_grid) or "default"; the fine halos as
    the smoother leaves them.  fields: parameters that are not options (outflowLinearExtrapol, reserved, mgBoundCorr)"""
    from oracle.pyoracle import Oracle

    import util

    if layout == "polar":
        import meshes

        prm = util.make_params(options)
        fine = meshes.polar_grid(*shape, prm, seed=seed)
    else:
        faces = {"inout": INOUT, "supin": SUPIN}.get(layout, (syn.IMIN, syn.IMAX, syn.JMIN, syn.JMAX, syn.KMIN, syn.KMAX))
        split = {"mixed": util.MIXED, "many": util.MANY}.get(layout)
        prm, fine = util.case(*shape, options, seed=seed, split=split, physical_faces=faces)
    for k, v in (fields or {}).items():
        setattr(prm, k, v)
    fine.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (syn.BC_WALL, 6) else 1)
    o = Oracle(fine, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    return prm, coarse_levels(fine, prm, nlev)[0]
