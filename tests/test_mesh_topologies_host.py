"""The O-grid, polar and axis-permuted test meshes of tests/meshes.py: their geometry, the periodic cut, the permutation
helper, and how far the oracle's own residual and time step move under an axis permutation (the bound the device
equivariance test in test_mesh_topologies_gpu.py is held to, times ten)."""
import numpy as np
import pytest

from adflow_b200 import make_params
from adflow_b200.halo import exchange_numpy
from oracle.pyoracle import Oracle

import meshes
from util import oracle_residual, rel_max

# Largest relative max-norm change of any dw row (owned cells, residual core, every discretisation) and of dtl that a
# cyclic axis permutation causes in the oracle on the blocks below, measured: 2.3e-14 (matrix dissipation on the polar
# grid, 5e-15 otherwise) and 3.7e-16.  The face sums of the sweeps run in i, j, k order, so a permutation reorders
# additions; nothing else may change.
ORACLE_EQUIVARIANCE_DW = 3e-14
ORACLE_EQUIVARIANCE_DTL = 1e-15

DISCS = ["central plus scalar dissipation", "central plus matrix dissipation", "upwind"]


def blocks(eq="RANS"):
    prm = make_params({"equationType": eq})
    o = meshes.o_grid(10, 12, 8, prm)
    return prm, {"o_grid": o, "polar": meshes.polar_grid(10, 12, 8, prm),
                 "o_grid_jk": meshes.permute_axes(o, (1, 2, 0)), "o_grid_ki": meshes.permute_axes(o, (2, 0, 1))}


CUT_AXIS = {"o_grid": 1, "polar": 1, "o_grid_jk": 0, "o_grid_ki": 2}


def _along(axis, idx):
    sl = [slice(None)] * 3
    sl[axis] = idx
    return tuple(sl)


@pytest.mark.parametrize("eq", ["Euler", "RANS"])
@pytest.mark.parametrize("name", list(CUT_AXIS))
def test_geometry(eq, name):
    prm, bl = blocks(eq)
    hb = bl[name]
    d = hb.d
    ow = d.owned()
    assert (hb.vol[ow] > 0).all()
    # closed cells: the six face vectors of every owned cell sum to zero
    I, J, K = slice(2, d.il + 1), slice(2, d.jl + 1), slice(2, d.kl + 1)
    s = (hb.si[2:d.il + 1, J, K] - hb.si[1:d.il, J, K] + hb.sj[I, 2:d.jl + 1, K] - hb.sj[I, 1:d.jl, K]
         + hb.sk[I, J, 2:d.kl + 1] - hb.sk[I, J, 1:d.kl])
    assert np.abs(s).max() < 1e-15 * max(np.abs(a).max() for a in (hb.si, hb.sj, hb.sk))
    # the haloCellRatio repair of the reference (preprocessingAPI.F90:3031-3064) never triggers on these blocks
    c = [slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1)]
    for a, (lo, hi, e, l_) in enumerate(((1, 2, d.ie, d.il), (1, 2, d.je, d.jl), (1, 2, d.ke, d.kl))):
        for h, o in ((lo, hi), (e, l_)):
            s1, s2 = list(c), list(c)
            s1[a], s2[a] = h, o
            assert (hb.vol[tuple(s1)] / hb.vol[tuple(s2)] > 1e-10).all()
    # the halo cells across the cut are their donors, geometry and state, bit for bit
    ax = CUT_AXIS[name]
    n, e, b = (d.nx, d.ny, d.nz)[ax], (d.ie, d.je, d.ke)[ax], (d.ib, d.jb, d.kb)[ax]
    for h, dn in ((1, n + 1), (e, 2)):
        assert np.array_equal(hb.vol[_along(ax, h)], hb.vol[_along(ax, dn)])
    for h, dn in ((0, n), (b, 3), (1, n + 1), (e, 2)):
        for arr in meshes.state_vars(hb):
            assert np.array_equal(arr[_along(ax, h)], arr[_along(ax, dn)])
    s_cut = (hb.si, hb.sj, hb.sk)[ax]
    for h, dn in ((0, n), (1, n + 1), (e, 2)):
        assert np.array_equal(s_cut[_along(ax, h)], s_cut[_along(ax, dn)])
    for s_other in [(hb.si, hb.sj, hb.sk)[q] for q in range(3) if q != ax]:
        assert np.array_equal(s_other[_along(ax, 1)], s_other[_along(ax, n + 1)])
        assert np.array_equal(s_other[_along(ax, e)], s_other[_along(ax, 2)])


def test_polar_axis():
    """kMin collapsed: every face vector on the axis is exactly 0, the halo nodes beyond it are the extrapolation of xhalo
    (x0 = 2 x1 - x2), i.e. the second node ring turned by pi about the axis, and the BCData normal is 0 there"""
    prm, bl = blocks()
    hb = bl["polar"]
    d = hb.d
    assert np.array_equal(hb.sk[1:d.ie + 1, 1:d.je + 1, 1], np.zeros((d.ie, d.je, 3)))
    assert (np.abs(hb.sk[2:d.il + 1, 2:d.jl + 1, 2]).sum(-1) > 0).all()
    x = hb.x
    assert np.array_equal(x[1:d.il + 1, :d.je + 1, 1, 1:], np.zeros((d.il, d.je + 1, 2)))
    assert np.array_equal(x[:, :d.je + 1, 0][:d.ie + 1], 2.0 * x[:d.ie + 1, :d.je + 1, 1] - x[:d.ie + 1, :d.je + 1, 2])
    np.testing.assert_allclose(x[1:d.il + 1, 1:d.jl + 1, 0, 1:], -x[1:d.il + 1, 1:d.jl + 1, 2, 1:], rtol=0, atol=1e-15)
    polar = [s for s in hb.subfaces if s["bcType"] == meshes.BC_SYMMPOLAR]
    assert len(polar) == 1 and polar[0]["faceId"] == 5 and not np.abs(polar[0]["norm"]).any()
    # the wedge cells next to the axis carry a residual of their own (not a negligible corner of the block)
    ho = oracle_residual(prm, hb)
    ow = d.owned()
    for l in range(hb.nw):
        assert np.isfinite(ho.dw[ow + (l,)]).all()
        assert np.abs(ho.dw[2:d.il + 1, 2:d.jl + 1, 2, l]).max() > 1e-3 * np.abs(ho.dw[ow + (l,)]).max()


def test_pattern_lists():
    prm, bl = blocks()
    hb = bl["o_grid"]
    d = hb.d
    p2, p1 = meshes.self_periodic_pattern(hb, 2), meshes.self_periodic_pattern(hb, 1)
    assert len(p2["haloList"]) == 4 * (d.ib + 1) * (d.kb + 1) and len(p1["haloList"]) == 2 * d.ie * d.ke
    for p in (p1, p2):
        h, dn = p["haloList"], p["donorList"]
        assert (h[:, 0] == 0).all() and (dn[:, 0] == 0).all()
        assert np.array_equal(h[:, [1, 3]], dn[:, [1, 3]])
        assert set(dn[:, 2].tolist()) <= {2, 3, d.ny, d.jl}          # donors are owned in j
        assert len({tuple(r) for r in h.tolist()}) == len(h)
    # the exchange is idempotent on the blocks handed out: their state already went through it once
    h2 = hb.copy()
    exchange_numpy([h2], p2, meshes.state_vars)
    for a, b in zip(meshes.state_vars(h2), meshes.state_vars(hb)):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("perm", meshes.CYCLIC[1:])
def test_permutation_round_trip(perm):
    """the permutation applied three times gives back the block, every array and subface bit for bit"""
    from adflow_b200 import synthetic as syn

    prm, bl = blocks()
    hb = bl["o_grid"]
    crs = syn.make_coarse_block(hb, prm)          # hb now carries interpolation tables too
    h3, c3 = hb, crs
    for _ in range(3):
        h3, c3 = meshes.permute_axes(h3, perm), meshes.permute_axes(c3, perm)
    for a, b in ((h3, hb), (c3, crs)):
        for name in ["w", "dw", "iblank", "porI", "porJ", "porK"] + a.REAL + a.VEC:
            assert np.array_equal(getattr(a, name), getattr(b, name)), name
        assert sorted(a.mg) == sorted(b.mg) and all(np.array_equal(a.mg[k], b.mg[k]) for k in b.mg)
        assert len(a.subfaces) == len(b.subfaces)
        for s, t in zip(a.subfaces, b.subfaces):
            assert sorted(s) == sorted(t)
            for k in s:
                assert np.array_equal(s[k], t[k]), k
    # one permutation: the metrics the blockette formula makes from the permuted nodes are the permuted metrics
    hp = meshes.permute_axes(hb, perm)
    h2 = hp.copy()
    syn.compute_metrics(h2)
    syn.compute_volumes(h2)
    for n in ("si", "sj", "sk", "vol"):
        a, b = getattr(h2, n), getattr(hp, n)
        assert np.abs(a - b).max() <= 1e-15 * np.abs(b).max(), n
    # and a subface's data sits over the same cells: the face's normal is the unit face vector again
    for s in hp.subfaces:
        if s["bcType"] == meshes.BC_SYMMPOLAR:
            continue
        t = syn.make_subface(hp, s["faceId"], s["bcType"], prm)
        assert np.abs(t["norm"] - s["norm"]).max() < 1e-15


@pytest.mark.parametrize("disc", DISCS)
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
def test_oracle_equivariance_bound(disc, eq):
    prm = make_params({"equationType": eq, "discretization": disc})
    for hb in (meshes.o_grid(10, 12, 8, prm), meshes.polar_grid(10, 12, 8, prm)):
        ow = hb.d.owned()
        ref = oracle_residual(prm, hb)
        ht = hb.copy()
        Oracle(ht, prm).time_step(True)
        for perm in meshes.CYCLIC[1:]:
            hp = meshes.permute_axes(hb, perm)
            got = meshes.unpermute(oracle_residual(prm, hp).dw, perm)
            for l in range(hb.nw):
                assert rel_max(got[ow + (l,)], ref.dw[ow + (l,)]) <= ORACLE_EQUIVARIANCE_DW, (perm, l)
            Oracle(hp, prm).time_step(True)
            assert rel_max(meshes.unpermute(hp.dtl, perm)[ow], ht.dtl[ow]) <= ORACLE_EQUIVARIANCE_DTL, perm


def test_symmetry_face_halo_nodes():
    """xhalo mirrors the halo nodes of a symmetry face about the plane of its corner diagonals; on an i face of the O-grid
    those diagonals are parallel (node jl is node 1), so the nodes stay the extrapolation, as with a far-field face"""
    from adflow_b200 import synthetic as syn

    prm = make_params()
    a = meshes.o_grid(10, 12, 8, prm, i_faces=(syn.BC_SYMM, syn.BC_SYMM))
    b = meshes.o_grid(10, 12, 8, prm, i_faces=(syn.BC_FARFIELD, syn.BC_FARFIELD))
    assert np.array_equal(a.x, b.x)
    # a planar symmetry face whose diagonals span the plane: the halo nodes are the mirror images of the second layer
    hb = a.copy()
    d = hb.d
    x = hb.x.copy()
    x[:, :, :, 1] += 0.3 * x[:, :, :, 0] ** 2          # a curved axial spacing, so that extrapolation is not a mirror
    x[:, :, :, 0] = np.arange(d.box[0])[:, None, None] * 0.1 - 0.1
    meshes._xhalo(x, d, symm_faces=(syn.JMIN,))
    v1 = x[d.il, 1, d.kl] - x[1, 1, 1]
    v2 = x[d.il, 1, 1] - x[1, 1, d.kl]
    n = np.cross(v1, v2) / np.linalg.norm(np.cross(v1, v2))
    got = x[:d.ie + 1, 0, :d.ke + 1]
    x1, x2 = x[:d.ie + 1, 1, :d.ke + 1], x[:d.ie + 1, 2, :d.ke + 1]
    np.testing.assert_allclose(got, x2 + 2.0 * ((x1 - x2) @ n)[..., None] * n, rtol=0, atol=1e-14)
