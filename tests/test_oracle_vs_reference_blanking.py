"""Pins the oracle against the reference's own routines (translated Fortran -> C, oracle/_ref) where overset blanking
and face porosities steer them, bit for bit:

  surfaceIntegrations.F90  wallIntegrationFace, weighted by the surface iblank BCData%iblank, which the overset zipper
                           makes differ from the volume iblank of the first cell layer
  residuals.F90            residual_block (the fluxes.F90 block routines behind every smoother) with noFlux / boundFlux
                           planes in i, j and k and blanked cells, at rFil 1.0, 0.56, 0.44 with the persistent fw
  fluxes.F90               inviscidDissFluxScalarCoarse / MatrixCoarse with an interior noFlux plane on level 2

Every test also shows that its blanking or porosity changes what it compares."""
import numpy as np
import pytest

from adflow_b200 import synthetic as syn
from oracle import refblockette as rb
from util import MIXED, blank_wall_surfaces, case, coarse_interior_planes, overset_layout, split_faces, volume_weighted, wall_layer

pytestmark = pytest.mark.skipif(not rb.available(), reason="oracle/_ref/libblockette_ref.so not built")

IMIN, IMAX, JMIN, JMAX, KMIN, KMAX = 1, 2, 3, 4, 5, 6
SYMM, WALL, FAR, EULERWALL, EXTRAP, ISOWALL = 1, 2, 3, 4, 5, 6
# relative tolerance of the device wall forces against the oracle (tests/test_forces.py); the surface iblank must move
# the forces by more than 1e3 times it
FORCE_TOL = 1e-11
WALLS = {
    "adiabatic": ({"equationType": "RANS"}, {IMIN: WALL, IMAX: FAR, JMIN: FAR, JMAX: SYMM, KMIN: FAR, KMAX: WALL}),
    "isothermal": ({"equationType": "RANS"}, {IMIN: FAR, IMAX: ISOWALL, JMIN: WALL, JMAX: FAR, KMIN: SYMM, KMAX: FAR}),
    "euler": ({"equationType": "Euler"}, {IMIN: FAR, IMAX: FAR, JMIN: SYMM, JMAX: EULERWALL, KMIN: EULERWALL, KMAX: FAR}),
    "MIXED": ({"equationType": "RANS"}, None),
}


def _eq(a, b, what):
    assert np.array_equal(a, b), "%s differs: max abs %.3e" % (what, np.abs(a - b).max())


def blanked_wall_case(walls, shape=(12, 9, 10), seed=314):
    """a block of the WALLS layouts after the residual that stores the wall stresses, every wall blanked by
    blank_wall_surfaces; MIXED splits the faces first, so that wall pieces carry different parts of the pattern"""
    from oracle.pyoracle import Oracle

    opts, perm = WALLS[walls]
    if perm is None:
        prm, hb = case(*shape, opts, seed=seed, split=MIXED)
    else:
        prm, hb = case(*shape, opts, seed=seed, physical_faces=perm)
    hb.subfaces.sort(key=lambda s_: 0 if s_["bcType"] in (WALL, ISOWALL) else 1)
    blank_wall_surfaces(hb)
    o = Oracle(hb, prm)
    if prm.equations == 3:
        o.apply_turb_bc(True)
    o.apply_flow_bc(True)
    o.residual_core(8 | (16 if prm.equations == 3 else 0))      # stores hb.wallTau
    return prm, hb


def forces_sensitivity(prm, hb, got, scale, ref_point, p_ref):
    """the surface iblank moves every nonzero row of the forces by more than 1e3 FORCE_TOL of its scale"""
    from oracle.pyoracle import Oracle

    hv = hb.copy()
    hv.subfaces = volume_weighted(hb)
    vol = Oracle(hv, prm).wall_forces(ref_point, p_ref)
    rows = scale[:, 0] > 0
    moved = np.abs(got - vol).max(axis=1)
    assert (moved[rows] > 1e3 * FORCE_TOL * scale[rows, 0]).all(), moved / np.where(scale[:, 0] > 0, scale[:, 0], 1)


@pytest.mark.parametrize("walls", list(WALLS))
def test_wall_forces_weighted_by_surface_iblank(walls):
    from oracle.pyoracle import Oracle

    prm, hb = blanked_wall_case(walls)
    nwall = 0
    for s in hb.subfaces:
        if s["bcType"] in (WALL, EULERWALL, ISOWALL):
            nwall += 1
            surf, vol = s["iblank"], hb.iblank[wall_layer(hb, s)]
            d = hb.d
            la = {1: d.jl, 2: d.jl, 3: d.il, 4: d.il, 5: d.il, 6: d.il}[s["faceId"]]
            lb = {1: d.kl, 2: d.kl, 3: d.kl, 4: d.kl, 5: d.jl, 6: d.jl}[s["faceId"]]
            own = (slice(max(2, s["icBeg"]) - s["icBeg"], min(la, s["icEnd"]) - s["icBeg"] + 1),
                   slice(max(2, s["jcBeg"]) - s["jcBeg"], min(lb, s["jcEnd"]) - s["jcBeg"] + 1))
            surf, vol = surf[own], vol[own]
            for sv, vv in ((1, -1), (0, 1), (-2, None), (0, 0)):        # the zipper's four kinds, on owned face cells
                hit = (surf == sv) if vv is None else (surf == sv) & (vol == vv)
                assert hit.any(), (s["faceId"], sv, vv)
    assert nwall >= (3 if walls == "MIXED" else 1)
    ref_point, p_ref = (0.3, -0.2, 0.1), 2.5
    mine = Oracle(hb, prm).wall_forces(ref_point, p_ref)
    ref = rb.wall_forces(hb, prm, ref_point, p_ref)
    _eq(mine, ref, "forces")
    scale = np.abs(mine).max(axis=1, keepdims=True)
    assert scale[0, 0] > 0 and (scale[1, 0] > 0) == (prm.equations != 1)
    forces_sensitivity(prm, hb, mine, scale, ref_point, p_ref)


def test_split_faces_slice_the_surface_iblank():
    prm, hb = case(12, 9, 10, {"equationType": "RANS"})
    blank_wall_surfaces(hb)
    whole = next(s for s in hb.subfaces if s["faceId"] == KMIN)["iblank"].copy()
    split_faces(hb, prm, {KMIN: MIXED[KMIN]})
    pieces = [s for s in hb.subfaces if s["faceId"] == KMIN]
    assert len(pieces) == 3
    for s in pieces:
        _eq(s["iblank"], whole[s["icBeg"] - 1:s["icEnd"], s["jcBeg"] - 1:s["jcEnd"]], "piece %d:%d" % (s["icBeg"], s["icEnd"]))
        assert s["iblank"].flags.f_contiguous and s["iblank"].dtype == np.int32


# ---------------------------------------------------------------------------------------------------------------------
# residual_block with porosities and blanking
DISCS = {"scalar": "central plus scalar dissipation", "matrix": "central plus matrix dissipation", "upwind": "upwind"}


def _block_residual_stages(hb, prm, stages):
    """oracle and reference residual_block over `stages` with the persistent fw; (dw, fw) owned per stage of both"""
    from oracle.pyoracle import Oracle

    ho = hb.copy()
    o = Oracle(ho, prm)
    ow = hb.d.owned()
    out = []
    for n, stage in enumerate(stages):
        o.residual_block(prm.cdisRK[stage])
        if n == 0:
            r = rb.call(hb, prm, "residuals_initres_block", 1, 5, 1, 1, rkstage=stage)
        else:
            rb.set_int("rkstage", stage)
            r = rb.again("residuals_initres_block", 1, 5, 1, 1)
        r = rb.again("residuals_residual_block")
        out.append(((ho.dw[ow][..., :5].copy(), ho.fw[ow].copy()), (r.a["dw"][ow][..., :5].copy(), r.a["fw"][ow].copy())))
    return out


@pytest.mark.parametrize("disc", list(DISCS))
@pytest.mark.parametrize("eq", ["RANS", "laminar NS"])
def test_block_residual_with_porosities_and_blanking(disc, eq):
    """rFil = cdisRK 1.0, 0.56, 0.44 of the 5-stage scheme, fw carried from stage to stage"""
    from oracle.pyoracle import Oracle

    prm, hb = case(12, 10, 9, {"equationType": eq, "discretization": DISCS[disc], "nRKStages": 5})
    Oracle(hb, prm).time_step(True)
    hb.fw[...] = 0.0
    plain = hb.copy()
    overset_layout(hb, at=(6, 4, 4))
    stages = [st for st in range(5) if prm.cdisRK[st] != 0.0]
    assert [prm.cdisRK[st] for st in stages] == [1.0, 0.56, 0.44]
    got = _block_residual_stages(hb, prm, stages)
    base = _block_residual_stages(plain, prm, stages)
    for st, ((dw, fw), (rdw, rfw)), ((dw0, fw0), _) in zip(stages, got, base):
        _eq(dw, rdw, "stage %d dw" % st)
        _eq(fw, rfw, "stage %d fw" % st)
        for a, a0, what in ((dw, dw0, "dw"), (fw, fw0, "fw")):
            moved = np.linalg.norm((a - a0).ravel()) / np.linalg.norm(a0.ravel())
            assert moved > 1e3 * 1e-12, (st, what, moved)
    ib = hb.iblank[hb.d.owned()]
    dw, fw = got[-1][0]
    assert (dw[ib <= 0] == 0).all() and np.abs(dw[ib == 1]).max() > 0


# ---------------------------------------------------------------------------------------------------------------------
# coarse-level residual_block with interior noFlux / boundFlux planes
@pytest.mark.parametrize("coarse_disc", ["scalar", "matrix"])
def test_coarse_residual_block_with_interior_planes(coarse_disc):
    """initres_block + residual_block on level 2 (dw from the forcing term wr, central fluxes with the porosities,
    inviscidDissFluxScalarCoarse / MatrixCoarse reading them as ppor, the fw blend) at rFil 1.0, 0.56, 0.44 with fw
    carried from stage to stage: the coarse block has the boundFlux wall faces of setPorosities and one interior plane
    of each direction, noFlux on part of it.  The reference keeps the coarse dw and fw in the finest level's arrays."""
    from oracle.pyoracle import Oracle
    from test_oracle_vs_reference_mg import oracle_transfer_to_coarse, two_levels

    def run(with_planes):
        prm, fine, coarse = two_levels((12, 8, 10), {"coarseDiscretization": DISCS[coarse_disc], "nRKStages": 5})
        if with_planes:
            coarse_interior_planes(coarse)
        oracle_transfer_to_coarse(prm, fine, coarse)
        # off the restricted state, as after a smoothing step: at w = w1 the forcing term cancels the coarse operator and
        # dw is the restricted fine residual whatever the coarse porosities
        ow = coarse.d.owned()
        coarse.w[ow + (slice(0, 5),)] *= 1.0 + 1e-3 * np.random.default_rng(4).standard_normal(coarse.w[ow + (slice(0, 5),)].shape)
        Oracle(coarse, prm).pressure(False)
        Oracle(coarse, prm).apply_flow_bc(False)
        coarse.fw[...] = 0.0
        stages = [st for st in range(5) if prm.cdisRK[st] != 0.0]
        assert [prm.cdisRK[st] for st in stages] == [1.0, 0.56, 0.44]
        mg = rb.RefMG(fine.copy(), coarse.copy(), prm)
        oc = Oracle(coarse, prm)
        out = []
        try:
            mg.seed_coarse_shared()
            for st in stages:
                mg.call(2, "residuals_initres_block", 1, 5, 2, 1, rkstage=st)
                mg.call(2, "residuals_residual_block", rkstage=st)
                oc.residual_block(prm.cdisRK[st])
                rf = mg.lv[1].a
                out.append(((coarse.dw[ow][..., :5].copy(), coarse.fw[ow].copy()),
                            (rf["dw"][ow][..., :5].copy(), rf["fw"][ow].copy())))
        finally:
            mg.close()
        return out

    got, base = run(True), run(False)
    for st, ((dw, fw), (rdw, rfw)), ((dw0, fw0), _) in zip((0, 2, 4), got, base):
        _eq(dw, rdw, "stage %d dw" % st)
        _eq(fw, rfw, "stage %d fw" % st)
        for a, a0, what in ((dw, dw0, "dw"), (fw, fw0, "fw")):
            moved = np.linalg.norm((a - a0).ravel()) / np.linalg.norm(a0.ravel())
            assert moved > 1e3 * 1e-12, (st, what, moved)
