"""Shared helpers for the parity tests (oracle = checker, CUDA path = product)."""
import numpy as np

from adflow_b200 import make_params
from adflow_b200 import synthetic as syn

FLOW, TURB, SKIP = 8, 16, 64


def rel_l2(a, b):
    """||a-b||_2 / ||b||_2 (SURVEY 8d: L2 norm of the dw difference / L2 norm of dw)."""
    nb = np.linalg.norm(b.ravel())
    return np.linalg.norm((a - b).ravel()) / (nb if nb > 0 else 1.0)


def rel_max(a, b):
    mb = np.abs(b).max()
    return np.abs(a - b).max() / (mb if mb > 0 else 1.0)


def case(nx, ny, nz, options=None, seed=314, split=None, **kw):
    """a synthetic block and its parameters; split: a layout for split_faces"""
    prm = make_params(options)
    hb = syn.make_block(nx, ny, nz, prm, seed=seed, **kw)
    if split:
        split_faces(hb, prm, split)
    return prm, hb


def split_faces(hb, prm, spec):
    """Replace the subface of every face named in spec by pieces along one in-plane direction.

    spec: face -> (direction, bcTypes, cuts).  direction 0 cuts the icBeg:icEnd range, 1 the jcBeg:jcEnd range; piece q
    has bcTypes[q], and pieces q and q+1 meet at [.., cuts[q]] | [cuts[q] + 1, ..].  Only block edges are halo-extended
    (the first piece starts at 1, the last ends at ie / je / ke).  A piece's prescribed data is that of a whole-face
    subface of its bcType, sliced to the piece, and so is the whole subface's surface iblank when it has one.  Viscous
    pieces go first, as the reference numbers them; porosities stay as the block was built."""
    subs = []
    for whole in hb.subfaces:
        if whole["faceId"] not in spec:
            subs.append(whole)
            continue
        axis, bcs, cuts = spec[whole["faceId"]]
        key = "jc" if axis else "ic"
        for bc, lo, hi in zip(bcs, [1] + [c + 1 for c in cuts], cuts + [whole[key + "End"]]):
            if prm.equations == syn.EULER and bc in (syn.BC_WALL, 6):
                bc = syn.BC_EULERWALL
            sub = syn.make_subface(hb, whole["faceId"], bc, prm, iblank=whole.get("iblank"))
            for k, v in sub.items():
                if isinstance(v, np.ndarray):
                    sub[k] = np.asfortranarray(v[:, lo - 1:hi] if axis else v[lo - 1:hi])
            sub[key + "Beg"], sub[key + "End"] = lo, hi
            subs.append(sub)
    hb.subfaces = sorted(subs, key=lambda s: 0 if s["bcType"] in (syn.BC_WALL, 6) else 1)


_SYMM, _WALL, _FAR, _EXTRAP, _ISOWALL, _SUBOUT, _SUBIN = 1, 2, 3, 5, 6, 7, 8
# Split-face layouts for split_faces, for blocks of at least 8 x 7 x 9 cells.  The cuts along k (the second in-plane
# direction of the i and j faces) avoid k = 1 mod 4, so they fall inside the planes of a form-function slab.
# MIXED: every face in two or three pieces, the BC class changing along the face.
MIXED = {syn.IMIN: (1, [_FAR, _WALL], [2]), syn.IMAX: (1, [_SUBIN, _SUBOUT], [7]),
         syn.JMIN: (1, [_SYMM, _FAR], [4]), syn.JMAX: (1, [_FAR, _ISOWALL, _FAR], [3, 8]),
         syn.KMIN: (0, [_WALL, _WALL, _FAR], [4, 7]), syn.KMAX: (1, [_EXTRAP, _FAR], [5])}
# MANY: five far-field pieces along k on both i faces, 14 subfaces in all: more than one launch of the SA wall terms
# carries (ADFB_BC_MAXSUB), and ten independent items in one level of the BC sweep, more than one launch carries
# (ADFB_BC_LEVEL_MAX).
# In both, a level of the sweep holds pieces of different lengths, the longest not first.
MANY = {syn.IMIN: (1, [_FAR] * 5, [2, 3, 4, 6]), syn.IMAX: (1, [_FAR] * 5, [2, 3, 4, 6])}


NOFLUX, BOUNDFLUX = -1, 0


def overset_layout(hb, at=(5, 5, 5)):
    """Blanking and face porosities of a block of an overset mesh (SURVEY C4), in place.

    at = (i, j, k): a fringe shell (iblank -1) over cells at-1 .. at+4 of each direction around a hole (0) at at+1 .. at+2,
    so that face `at` of each direction lies between fringe and hole (both clipped to the owned cells); on those three
    faces, noFlux on the cells below the middle of the plane and boundFlux above it.  A fringe slab two cells deep along
    jMax, and holes in the first cell layer of kMin (the wall face of the default layout).  Owned cells only; the faces
    `at` must be interior faces."""
    d = hb.d
    i, j, k = at
    assert 2 <= i < d.il and 2 <= j < d.jl and 2 <= k < d.kl, (at, d.il, d.jl, d.kl)
    ow = d.owned()

    def box(a, lo, hi, l_):
        return slice(max(2, a + lo), min(l_, a + hi) + 1)

    hb.iblank[box(i, -1, 4, d.il), box(j, -1, 4, d.jl), box(k, -1, 4, d.kl)] = -1
    hb.iblank[box(i, 1, 2, d.il), box(j, 1, 2, d.jl), box(k, 1, 2, d.kl)] = 0
    hb.iblank[2:d.il + 1, d.jl - 1:d.jl + 1, 2:d.kl + 1] = -1
    hb.iblank[2:5, 2:4, 2] = 0
    hb.iblank[d.il - 1, 3, 2] = 0
    jm, km, im = (d.jl + 2) // 2, (d.kl + 2) // 2, (d.il + 2) // 2
    hb.porI[i, 2:jm, 2:d.kl + 1] = NOFLUX
    hb.porI[i, jm:d.jl + 1, 2:d.kl + 1] = BOUNDFLUX
    hb.porJ[2:d.il + 1, j, 2:km] = NOFLUX
    hb.porJ[2:d.il + 1, j, km:d.kl + 1] = BOUNDFLUX
    hb.porK[2:im, 2:d.jl + 1, k] = NOFLUX
    hb.porK[im:d.il + 1, 2:d.jl + 1, k] = BOUNDFLUX
    assert (hb.iblank[ow] == 0).any() and (hb.iblank[ow] == -1).any() and (hb.iblank[ow] == 1).any()
    return hb


def coarse_interior_planes(hb):
    """porosities of a coarse multigrid block: the boundFlux faces setPorosities gave it, plus one interior plane in each
    direction, noFlux on the cells below the middle of the plane and boundFlux above it"""
    d = hb.d
    fi, fj, fk = (min(3, l_ - 1) for l_ in (d.il, d.jl, d.kl))
    jm, km, im = (d.jl + 2) // 2, (d.kl + 2) // 2, (d.il + 2) // 2
    hb.porI[fi, 2:jm, 2:d.kl + 1], hb.porI[fi, jm:d.jl + 1, 2:d.kl + 1] = NOFLUX, BOUNDFLUX
    hb.porJ[2:d.il + 1, fj, 2:km], hb.porJ[2:d.il + 1, fj, km:d.kl + 1] = NOFLUX, BOUNDFLUX
    hb.porK[2:im, 2:d.jl + 1, fk], hb.porK[im:d.il + 1, 2:d.jl + 1, fk] = NOFLUX, BOUNDFLUX
    return hb


WALL_BCS = (syn.BC_WALL, syn.BC_EULERWALL, 6)


def wall_layer(hb, s):
    """index of the first interior cell layer under subface s, over its cell range icBeg:icEnd x jcBeg:jcEnd"""
    d = hb.d
    sl = [slice(s["icBeg"], s["icEnd"] + 1), slice(s["jcBeg"], s["jcEnd"] + 1)]
    sl.insert((s["faceId"] - 1) // 2, {1: 2, 2: d.il, 3: 2, 4: d.jl, 5: 2, 6: d.kl}[s["faceId"]])
    return tuple(sl)


def blank_wall_surfaces(hb):
    """Give every wall subface a surface iblank (BCData%iblank) that differs from the volume iblank of the first cell
    layer in the four ways the overset zipper makes it differ, in a pattern over the face's cell indices: volume -1 and
    surface 1 (a fringe restored by slit elimination), volume 1 and surface 0 (surface priority), surface -2 (a forced
    receive, volume -1), volume 0 and surface 0 (a hole); both 1 elsewhere."""
    for s in hb.subfaces:
        if s["bcType"] not in WALL_BCS:
            continue
        a, b = np.meshgrid(np.arange(s["icBeg"], s["icEnd"] + 1), np.arange(s["jcBeg"], s["jcEnd"] + 1), indexing="ij")
        code = (a + 2 * b) % 6
        s["iblank"] = np.asfortranarray(np.select([code == 1, code == 2, code == 3], [0, -2, 0], 1), dtype=np.int32)
        hb.iblank[wall_layer(hb, s)] = np.select([code == 0, code == 2, code == 3], [-1, -1, 0], 1)


def volume_weighted(hb):
    """hb's subfaces with the surface iblank of every wall replaced by the volume iblank of the first cell layer: the
    weighting wall forces had before they read BCData%iblank"""
    subs = []
    for s in hb.subfaces:
        s = dict(s)
        if s["bcType"] in WALL_BCS:
            s["iblank"] = np.asfortranarray(hb.iblank[wall_layer(hb, s)], dtype=np.int32)
        subs.append(s)
    return subs


def oracle_residual(prm, hb, flags=FLOW | TURB, rfil=1.0):
    from oracle.pyoracle import Oracle

    ho = hb.copy()
    Oracle(ho, prm).residual_core(flags, rfil)
    return ho


def oracle_form_function(prm, hb, wvec):
    """FormFunction_mf on one block with the oracle: setW (turbulence clip), blocketteRes
    (p/rlv/rev, BCs, whalo2's owned-cell etot, core), setRVec."""
    import ctypes as C

    from oracle.pyoracle import Oracle

    d = hb.d
    ow = d.owned()
    h2 = hb.copy()
    v = np.asarray(wvec).reshape(d.nz, d.ny, d.nx, hb.nw).transpose(2, 1, 0, 3).copy()
    if hb.nw > 5:
        v[..., 5] = np.maximum(1e-6 * prm.wInf[5], v[..., 5])
    h2.w[ow] = v
    o = Oracle(h2, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(FLOW | TURB)
    r = h2.dw[ow] / h2.volRef[ow][..., None]
    if hb.nw > 5:
        r[..., 5] *= prm.turbResScale
    return np.transpose(r, (2, 1, 0, 3)).reshape(-1)
