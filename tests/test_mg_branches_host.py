"""Each multigrid branch tests/test_mg_boundaries_gpu.py holds the device to changes the result, on the oracle (no GPU):
a kernel that ignored the branch would fail there by far more than the tolerance (1e-9 on state changes)."""
import numpy as np

from oracle.pyoracle import Oracle

import fmg_oracle as fo
import mg_coarsen as mc
from test_mg_gpu import oracle_transfer_to_coarse
from util import rel_max, wall_layer

MARGIN = 1e3 * 1e-9
LIN = {"viscWallTreatment": "linear pressure extrapolation"}


def fmg_ground_states(options):
    prm, lv = mc.layout_levels("inout", (12, 9, 10), options, 3)
    oracle_transfer_to_coarse(prm, lv[0], lv[1])
    oracle_transfer_to_coarse(prm, lv[1], lv[2])
    for hb in lv:
        hb.fw[...] = 0
    return fo.full_multigrid_start_up(prm, lv, 3, 2, "3w")


def test_wall_pressure_treatment_matters_on_a_ground_level_only():
    """linear or constant pressure at the walls: ground level 2 of the start-up differs, a level above the ground
    level (constant pressure whatever is asked) is the same bit for bit"""
    lin, const = fmg_ground_states(LIN), fmg_ground_states(None)
    assert rel_max(lin[2][0], const[2][0]) > MARGIN, rel_max(lin[2][0], const[2][0])
    prm, lv = mc.layout_levels("inout", (12, 9, 10), None, 2)
    out = []
    for constant in (0, 1):
        prm.wallBCConstantPressure = constant
        fine, coarse = (hb.copy() for hb in lv)
        oracle_transfer_to_coarse(prm, fine, coarse)
        Oracle(coarse, prm).rk_smoother()
        out.append(coarse.w.copy())
    assert np.array_equal(out[0], out[1])


def prolonged(layout, neumann, shape):
    prm, (fine, coarse) = mc.layout_levels(layout, shape, None, 2, {"mgBoundCorr": neumann})
    oracle_transfer_to_coarse(prm, fine, coarse)
    Oracle(coarse, prm).rk_smoother()
    w0 = fine.w.copy()
    of = Oracle(fine, prm)
    of.mg_prolong(Oracle(coarse, prm))
    of.apply_flow_bc(True)
    return fine, w0


def test_boundary_correction_matters_next_to_every_non_symmetry_class():
    """mgBoundCorr 0 (zero corrections in the coarse halos) or 1 (Neumann): the prolonged fine state in the first
    cell layer under every non-symmetry subface moves by far more than the tolerance, relative to the state change"""
    seen = set()
    for layout, shape in (("inout", (12, 9, 10)), ("supin", (11, 10, 9)), ("polar", (10, 12, 8))):
        f0, w0 = prolonged(layout, 0, shape)
        f1, _ = prolonged(layout, 1, shape)
        change = np.abs(f0.w[f0.d.owned()][..., :5] - w0[f0.d.owned()][..., :5]).max()
        for s in f0.subfaces:
            if s["bcType"] == 1:
                continue
            lay = wall_layer(f0, s)
            moved = np.abs(f1.w[lay][..., :5] - f0.w[lay][..., :5]).max() / change
            assert moved > MARGIN, (layout, s["faceId"], s["bcType"], moved)
            seen.add(s["bcType"])
    assert seen == {2, 3, 5, 6, 7, 8, 9, 10, 11}


def test_an_irregular_min_end_cell_interpolates_with_itself():
    """mgICoarse of the fine cell of an irregular min-end coarse cell is (2, 2) (coarseUtils.F90:353-386): its
    prolongation reads no coarse halo, so the boundary correction leaves it alone in that direction, while the fine
    cell 2 of a regular min end interpolates with the halo and moves"""
    prm, lv = mc.layout_levels("inout", (12, 9, 10), None, 3)
    fine, coarse = lv[1], lv[2]                  # level 3 is right-started in j: irregular cell at the min end
    assert coarse.mg["mgJWeight"][2] == 0.5 and coarse.mg["mgIWeight"][2] == 1.0
    assert tuple(fine.mg["mgJCoarse"][2]) == (2, 2) and tuple(fine.mg["mgICoarse"][2]) == (2, 1)
    out = []
    for neumann in (0, 1):
        prm.mgBoundCorr = neumann
        l1, l2, l3 = (hb.copy() for hb in lv)
        oracle_transfer_to_coarse(prm, l1, l2)
        oracle_transfer_to_coarse(prm, l2, l3)
        Oracle(l3, prm).rk_smoother()
        Oracle(l2, prm).mg_prolong(Oracle(l3, prm))
        out.append(l2.w.copy())
    d = fine.d

    def interior(a):                             # fine cells whose interpolation partners are interior coarse cells
        c, l_ = fine.mg["mg%sCoarse" % "IJK"[a]], (d.il, d.jl, d.kl)[a]
        dc = coarse.d
        return [i for i in range(2, l_ + 1) if min(c[i]) >= 2 and max(c[i]) <= (dc.il, dc.jl, dc.kl)[a]]

    ii, jj, kk = interior(0), interior(1), interior(2)
    assert 2 in jj and 2 not in ii
    at_j = np.ix_(ii, [2], kk)
    assert np.array_equal(out[0][at_j], out[1][at_j])
    at_i = np.ix_([2], jj, kk)
    assert np.abs(out[0][at_i][..., :5] - out[1][at_i][..., :5]).max() > 0
