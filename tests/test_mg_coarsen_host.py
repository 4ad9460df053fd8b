"""The reference's coarsening of tests/mg_coarsen.py on the boundary layouts the multigrid tests run: what
createCoarseBlocks guarantees (subface ends kept, one or two fine cells per coarse cell, pieces that tile their face,
alternating start sides) and the irregular cells those layouts are chosen for."""
import numpy as np
import pytest

from adflow_b200 import synthetic as syn
from oracle.pyoracle import Oracle

import mg_coarsen as mc

LAYOUTS = [("inout", (12, 9, 10)), ("inout", (13, 9, 11)), ("supin", (11, 10, 9)), ("mixed", (12, 9, 10)),
           ("many", (11, 8, 9)), ("polar", (10, 12, 8)), ("default", (16, 12, 8))]


def kept(coarse, a):
    """fine nodes the coarse level of direction a keeps: node 1, then mgIFine(ii, 2) for ii = 2..il"""
    dc = coarse.d
    f = coarse.mg["mg%sFine" % "IJK"[a]]
    return np.concatenate([[1], f[2:(dc.il, dc.jl, dc.kl)[a] + 1, 1]])


@pytest.fixture(scope="module", params=LAYOUTS, ids=["%s-%dx%dx%d" % ((l,) + s) for l, s in LAYOUTS])
def levels(request):
    layout, shape = request.param
    return mc.layout_levels(layout, shape, nlev=3)


def test_subface_end_nodes_are_kept(levels):
    prm, lv = levels
    for fine, coarse in zip(lv, lv[1:]):
        for s in fine.subfaces:
            for a, (b, e) in enumerate(mc.node_ranges(fine, s)):
                assert {b, e} <= set(kept(coarse, a)), (s["faceId"], s["bcType"], a, b, e)


def test_every_coarse_cell_holds_one_or_two_fine_cells(levels):
    prm, lv = levels
    for fine, coarse in zip(lv, lv[1:]):
        df, dc = fine.d, coarse.d
        for a in range(3):
            nm = "IJK"[a]
            lf, lc = (df.il, df.jl, df.kl)[a], (dc.il, dc.jl, dc.kl)[a]
            f, w = coarse.mg["mg%sFine" % nm], coarse.mg["mg%sWeight" % nm]
            cells = []
            for ii in range(2, lc + 1):
                n = f[ii, 1] - f[ii, 0] + 1
                assert n in (1, 2) and w[ii] == (0.5 if n == 1 else 1.0), (nm, ii, f[ii], w[ii])
                cells += list(range(f[ii, 0], f[ii, 1] + 1))
            assert cells == list(range(2, lf + 1)), nm
            # mgICoarse: the coarse cell of every fine cell and the neighbour it interpolates with
            c = fine.mg["mg%sCoarse" % nm]
            for ii in range(2, lc + 1):
                for i in range(f[ii, 0], f[ii, 1] + 1):
                    assert c[i, 0] == ii and abs(c[i, 1] - ii) <= 1, (nm, i, c[i])


def test_the_pieces_of_a_face_tile_the_coarse_face(levels):
    prm, lv = levels
    for hb in lv:
        d = hb.d
        for face in range(1, 7):
            subs = [s for s in hb.subfaces if s["faceId"] == face]
            if not subs:
                continue
            a0, a1 = mc.IN_PLANE[face]
            e = (d.ie, d.je, d.ke)
            cover = np.zeros((e[a0] + 1, e[a1] + 1), dtype=int)
            for s in subs:
                cover[s["icBeg"]:s["icEnd"] + 1, s["jcBeg"]:s["jcEnd"] + 1] += 1
                na, nb = s["icEnd"] - s["icBeg"] + 1, s["jcEnd"] - s["jcBeg"] + 1
                assert s["norm"].shape == (na, nb, 3)
                for k, v in s.items():
                    if isinstance(v, np.ndarray) and k != "norm":
                        assert v.shape == (na, nb), (face, k)
            assert (cover[1:, 1:] == 1).all(), (hb.level, face)
        assert [s["bcType"] in (2, 6) for s in hb.subfaces] == sorted((s["bcType"] in (2, 6) for s in hb.subfaces), reverse=True)


def test_split_pieces_stay_split_on_every_level():
    prm, lv = mc.layout_levels("mixed", (12, 9, 10), nlev=3)
    n = [len(hb.subfaces) for hb in lv]
    assert n == [14] * 3
    for hb in lv[1:]:
        for s in hb.subfaces:
            assert s["icEnd"] >= s["icBeg"] and s["jcEnd"] >= s["jcBeg"]


def test_start_sides_alternate():
    """level 2 left-started; level 3 right-started in every direction level 2 did not halve"""
    prm, fine = mc.layout_levels("inout", (13, 9, 11), nlev=1)
    lv, coarsened = mc.coarse_levels(fine[0], prm, 3)
    assert coarsened[1] == (mc.LEFT, mc.LEFT, mc.LEFT)
    # k: 6 cells of level 2 right-started into 3, an exact halving, so level 3 counts as regular again
    assert coarsened[2] == (mc.RIGHT, mc.RIGHT, mc.REGULAR)
    # 13 cells: left-started keeps 1, 3, .., 13, 14 (irregular cell at the max end); right-started then keeps the max
    # end and every other node down from it, which leaves the irregular cell at the min end
    assert list(kept(lv[1], 0)) == [1, 3, 5, 7, 9, 11, 13, 14]
    assert list(kept(lv[2], 0)) == [1, 2, 4, 6, 8]
    assert lv[2].mg["mgIWeight"][2] == 0.5
    # a direction halved exactly is regular again, and the next level starts from the left
    prm, fine = mc.layout_levels("default", (16, 12, 8), nlev=1)
    lv, coarsened = mc.coarse_levels(fine[0], prm, 3)
    assert coarsened[1] == coarsened[2] == (mc.REGULAR,) * 3


def test_irregular_cells_inside_lines_and_at_min_ends():
    """the layouts of the multigrid tests put an irregular coarse cell inside a line (between two regular ones) and
    one at the min end of a line, where the prolongation reads the coarse halo"""
    inside = at_min = False
    for layout, shape in LAYOUTS:
        prm, lv = mc.layout_levels(layout, shape, nlev=3)
        for hb in lv[1:]:
            d = hb.d
            for a, nm in enumerate("IJK"):
                lc = (d.il, d.jl, d.kl)[a]
                irr = np.flatnonzero(hb.mg["mg%sWeight" % nm][2:lc + 1] == 0.5) + 2
                at_min |= 2 in irr
                inside |= any(2 < ii < lc for ii in irr)
    assert inside and at_min


def test_default_layout_coarsens_as_make_coarse_block():
    """whole faces and even cell counts: the reference's coarsening is synthetic.make_coarse_block's"""
    prm, lv = mc.layout_levels("default", (16, 12, 8), nlev=3)
    fine = lv[0].copy()
    b2 = syn.make_coarse_block(fine, prm)
    b3 = syn.make_coarse_block(b2, prm)
    for got, want in ((lv[1], b2), (lv[2], b3)):
        assert np.array_equal(got.x, want.x) and np.array_equal(got.vol, want.vol)
        for k in want.mg:
            assert np.array_equal(got.mg[k], want.mg[k]), k
        for n in ("porI", "porJ", "porK"):      # over the reference's bounds, the ones setPorosities sets
            sl = got.d.ref_slices(n)
            assert np.array_equal(getattr(got, n)[sl], getattr(want, n)[sl]), n


def test_restriction_of_a_uniform_state_returns_it():
    """the restriction of a uniform fine residual is, bit for bit, the number of fine cells each coarse cell holds
    (weight 1/2 on the doubled cell of an irregular direction); the volume-weighted restriction of a uniform state
    is that state to a few units in the last place -- the reference multiplies the volume-weighted sum by the
    reciprocal of the summed volume, which rounds"""
    for layout, shape in LAYOUTS:
        prm, lv = mc.layout_levels(layout, shape, nlev=3)
        for fine, coarse in zip(lv, lv[1:]):
            for l in range(5):
                fine.w[..., l] = (0.75, 0.25, -0.125, 0.0625, 2.5)[l]
            fine.p[...] = 1.0
            fine.rev[...] = 0.5
            fine.dw[...] = 1.0
            Oracle(coarse, prm).mg_restrict(Oracle(fine, prm))
            dc = coarse.d
            ow = dc.owned()
            n = [np.diff(coarse.mg["mg%sFine" % nm][2:l_ + 1], axis=1)[:, 0] + 1
                 for nm, l_ in zip("IJK", (dc.il, dc.jl, dc.kl))]
            cells = n[0][:, None, None] * n[1][None, :, None] * n[2][None, None, :]
            for l in range(5):
                assert np.array_equal(coarse.wr[ow][..., l], cells.astype(float)), (layout, coarse.level, l)
            for l in range(4):
                a, b = coarse.w[ow][..., l], fine.w[2, 2, 2, l]
                assert (np.abs(a - b) <= 4 * np.spacing(abs(b))).all(), (layout, coarse.level, l)
            assert (np.abs(coarse.p[ow] - 1.0) <= 4 * np.spacing(1.0)).all()
            assert (np.abs(coarse.rev[ow] - 0.5) <= 4 * np.spacing(0.5)).all()
