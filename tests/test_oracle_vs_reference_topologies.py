"""Pins the oracle against the reference's own routines (translated Fortran -> C, oracle/_ref) on the meshes of
tests/meshes.py: the O-grid, the polar grid with its collapsed kMin face, and the O-grid with its wall normal along j and
along i.  Bit-exact, like the other test_oracle_vs_reference_* files; the periodic cut is not exchanged here (setPointers
and whalo are stubs of the translated library), so these pin the per-block routines on this geometry: the residual core
with the 1e-25 floors of the radius ratios and of the upwind face areas, every BC including the polar one on a face of
zero area, the time step on wedge cells, the smoother stages, the SA block and the wall forces on curved walls."""
import numpy as np
import pytest

from adflow_b200 import make_params
from oracle import refblockette as rb
from oracle.pyoracle import Oracle

import meshes

pytestmark = pytest.mark.skipif(not rb.available(), reason="oracle/_ref/libblockette_ref.so not built")

FLOW, TURB, DISS_APPROX, VISC_APPROX = 8, 16, 1, 2
DISCS = ["central plus scalar dissipation", "central plus matrix dissipation", "upwind"]
BLOCKS = ["o_grid", "polar", "o_grid_jk", "o_grid_ki"]


def block(name, options=None):
    opts = {"equationType": "RANS"}
    opts.update(options or {})
    prm = make_params(opts)
    if name == "polar":
        return prm, meshes.polar_grid(10, 12, 8, prm)
    hb = meshes.o_grid(10, 12, 8, prm)
    perm = {"o_grid": (0, 1, 2), "o_grid_jk": (1, 2, 0), "o_grid_ki": (2, 0, 1)}[name]
    return prm, meshes.permute_axes(hb, perm)


def _eq(a, b, what):
    assert np.array_equal(a, b), "%s differs: max abs %.3e" % (what, np.abs(a - b).max())


@pytest.mark.parametrize("name", BLOCKS)
@pytest.mark.parametrize("disc", DISCS)
@pytest.mark.parametrize("flags", [0, DISS_APPROX | VISC_APPROX], ids=["exact", "approx"])
def test_residual_core(name, disc, flags):
    prm, hb = block(name, {"discretization": disc})
    Oracle(hb, prm).reference_shock_sensor()
    ho = hb.copy()
    Oracle(ho, prm).residual_core(FLOW | TURB | flags)
    r = rb.residual_core(hb, prm, FLOW | TURB | flags)
    ow = hb.d.owned()
    for l in range(hb.nw):
        assert np.abs(ho.dw[ow + (l,)]).max() > 0
        _eq(r.a["dw"][ow + (l,)], ho.dw[ow + (l,)], "dw[%d]" % l)


@pytest.mark.parametrize("name", BLOCKS)
@pytest.mark.parametrize("eq", ["Euler", "RANS"])
@pytest.mark.parametrize("second", [True, False])
def test_bcs(name, eq, second):
    prm, hb = block(name, {"equationType": eq})
    ho = hb.copy()
    Oracle(ho, prm).apply_flow_bc(second)
    r = rb.call(hb, prm, "bcroutines_applyallbc_block", int(second))
    for n in ("w", "p", "rlv", "rev"):
        _eq(r.a[n], getattr(ho, n), n)
    if eq == "RANS":
        ho = hb.copy()
        Oracle(ho, prm).apply_turb_bc(second)
        rb.call(hb, prm, "turbbcroutines_bcturbtreatment")
        r = rb.again("turbbcroutines_applyallturbbcthisblock", int(second))
        _eq(r.a["w"][..., 5], ho.w[..., 5], "nuTilde")
        _eq(r.a["rev"], ho.rev, "rev")


def test_polar_bc_moves_the_axis_halos():
    """the polar BC on the collapsed face writes both halo layers beyond the axis"""
    prm, hb = block("polar")
    ho = hb.copy()
    Oracle(ho, prm).apply_flow_bc(True)
    d = hb.d
    for k in (0, 1):
        assert not np.array_equal(ho.w[2:d.il + 1, 2:d.jl + 1, k], hb.w[2:d.il + 1, 2:d.jl + 1, k])


def _residual_state(name, options):
    prm, hb = block(name, options)
    o = Oracle(hb, prm)
    o.time_step(True)
    o.residual_block(1.0)
    hb.wn[...] = hb.w[..., :5]
    hb.pn[...] = hb.p
    return prm, hb


@pytest.mark.parametrize("name", BLOCKS)
@pytest.mark.parametrize("disc", DISCS)
def test_time_step(name, disc):
    prm, hb = block(name, {"discretization": disc})
    ho = hb.copy()
    Oracle(ho, prm).time_step(True)
    r = rb.call(hb, prm, "solverutils_timestep_block", 0)
    d = hb.d
    _eq(r.a["dtl"][d.owned()], ho.dtl[d.owned()], "dtl")
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    if disc == DISCS[0]:
        for ref, mine in (("radi", "radI"), ("radj", "radJ"), ("radk", "radK")):
            _eq(r.a[ref][c1], getattr(ho, mine)[c1], ref)


@pytest.mark.parametrize("name", BLOCKS)
@pytest.mark.parametrize("avg", ["never", "always"])
def test_rk_stage(name, avg):
    prm, hb = _residual_state(name, {"resAveraging": avg})
    ho = hb.copy()
    Oracle(ho, prm).rk_stage(2)
    r = rb.call(hb, prm, "smoothers_executerkstage", rkstage=2)
    _eq(r.a["w"][..., :5], ho.w[..., :5], "w")
    for n in ("p", "rlv", "rev"):
        _eq(r.a[n], getattr(ho, n), n)


@pytest.mark.parametrize("name", BLOCKS)
def test_dadi_step(name):
    prm, hb = _residual_state(name, {"smoother": "DADI"})
    ho = hb.copy()
    Oracle(ho, prm).dadi_step()
    r = rb.call(hb, prm, "smoothers_executedadistep", rkstage=0)
    _eq(r.a["w"][..., :5], ho.w[..., :5], "w")
    _eq(r.a["p"], ho.p, "p")


@pytest.mark.parametrize("name", BLOCKS)
def test_sa_block(name):
    prm, hb = block(name)
    ho = hb.copy()
    Oracle(ho, prm).sa_block()
    r = rb.call(hb, prm, "sa_sa_block", 0)
    ow = hb.d.owned()
    _eq(r.a["dw"][ow + (5,)], ho.dw[ow + (5,)], "dw(itu1)")
    _eq(r.a["w"][..., 5], ho.w[..., 5], "nuTilde")
    _eq(r.a["rev"], ho.rev, "rev")
    assert np.abs(ho.w[ow + (5,)] - hb.w[ow + (5,)]).max() > 0


@pytest.mark.parametrize("name", ["o_grid", "o_grid_jk", "o_grid_ki", "polar"])
def test_wall_forces(name):
    prm, hb = block(name)
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.residual_core(FLOW | TURB)
    ref_point = (0.3, -0.2, 0.1)
    mine = o.wall_forces(ref_point, p_ref=2.5)
    ref = rb.wall_forces(hb, prm, ref_point, p_ref=2.5)
    assert np.abs(mine[0]).max() > 0 and np.abs(mine[1]).max() > 0
    _eq(mine, ref, "forces")
