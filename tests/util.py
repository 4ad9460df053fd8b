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
    subface of its bcType, sliced to the piece.  Viscous pieces go first, as the reference numbers them; porosities
    stay as the block was built."""
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
            sub = syn.make_subface(hb, whole["faceId"], bc, prm)
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
