"""CUDA path against the oracle in the flow regimes of tests/regimes.py: contact discontinuities (JST sensor cap,
fourth difference cut off), a supersonic free stream with a subsonic pocket (both supersonic far-field branches,
one-signed eigenvalues), a stagnation slab (near-zero normal velocities, SA rr clip), the pressure floor of the state
preparation and the turbulence clip of setW, and far-field inflow and outflow on both j faces.  Every test first asserts
that its state reaches the branches it is about.  Also: the SA and DADI line solves at the line lengths where their
dispatch changes kernel.

Tolerances are those of the smooth-state parity files: 1e-12 on residuals, 1e-10 / 1e-9 on state changes over a
smoother cycle, 1e-13 on BC halos.  A jump cell's residual can be 100x the rest, so the cells more than two cells away
from a contact are also held to the residual tolerance on their own."""
import ctypes as C
import os

import numpy as np
import pytest

import regimes as R
from adflow_b200.solver import ADFLOW_B200, RES_DISS_APPROX, RES_FLOW, RES_SKIP_PREAMBLE, RES_TURB, RES_VISC_APPROX
from oracle.pyoracle import Oracle
from test_regimes_reach import assert_reaches
from util import oracle_form_function, oracle_residual, rel_l2, rel_max

pytestmark = pytest.mark.gpu

TOL = 1e-12
SHAPE = (12, 10, 8)
CONTACTS = ("contact_i", "contact_j", "contact_k")
SCALAR, MATRIX, UPWIND = ("central plus scalar dissipation", "central plus matrix dissipation", "upwind")


def _rows_close(hb, regime, got, want, rows, tol, at=None, what="dw"):
    ow = hb.d.owned()
    far = R.owned_away_from(hb, regime, at) if regime in CONTACTS else None
    for l in rows:
        a, b = got[ow + (l,)], want[ow + (l,)]
        assert np.isfinite(a).all(), (what, l)
        assert rel_l2(a, b) < tol, "%s[%d] rel L2 %.3e" % (what, l, rel_l2(a, b))
        assert rel_max(a, b) < 10 * tol, "%s[%d] rel max %.3e" % (what, l, rel_max(a, b))
        if far is not None:
            assert rel_max(a[far], b[far]) < 10 * tol, "%s[%d] away from the jump: rel max %.3e" % (what, l, rel_max(a[far], b[far]))


def _residual(prm, hb, flags):
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.residual(flags)
        return s.downloadResidual(0)
    finally:
        s.close()


def _sensor_keys(regime, disc):
    if disc == UPWIND or regime not in CONTACTS + ("supersonic",):
        return []
    pre = "matrix_sensor_cap_" if disc == MATRIX else "sensor_cap_"
    return [pre + a for a in ("ijk" if regime == "supersonic" else regime[-1])]


# ---------------------------------------------------------------------------------------------------------------------
# full residual
@pytest.mark.parametrize("regime", CONTACTS + ("supersonic", "stagnation", "low_reynolds"))
@pytest.mark.parametrize("eq,disc", [("RANS", SCALAR), ("laminar NS", SCALAR), ("RANS", MATRIX), ("RANS", UPWIND),
                                     ("Euler", UPWIND)])
def test_residual_in_regimes(cuda_lib, regime, eq, disc):
    if disc == MATRIX and regime in CONTACTS:
        pytest.skip("a contact at constant pressure does not reach the pressure sensor of matrix dissipation")
    if eq == "Euler" and regime == "low_reynolds":
        pytest.skip("the non-dimensional Euler state does not depend on the free-stream pressure")
    prm, hb = R.regime_case(regime, SHAPE, {"equationType": eq, "discretization": disc})
    keys = _sensor_keys(regime, disc) if eq != "Euler" else []
    keys += {"supersonic": ["supersonic_i"], "stagnation": ["stagnant_j"] + (["sa_rr_clip"] if eq == "RANS" else []),
             "low_reynolds": ["low_cell_re"]}.get(regime, [])
    assert_reaches(prm, hb, regime, keys)
    flags = RES_FLOW | (RES_TURB if eq == "RANS" else 0)
    ref = oracle_residual(prm, hb, flags)
    dw = _residual(prm, hb, flags | RES_SKIP_PREAMBLE)
    _rows_close(hb, regime, dw, ref.dw, range(hb.nw if eq == "RANS" else 5), TOL)


@pytest.mark.parametrize("regime", CONTACTS + ("supersonic",))
@pytest.mark.parametrize("seam", [0, 1])
def test_residual_with_jump_on_tile_and_chunk_seams(cuda_lib, regime, seam):
    """ADFB_TILE=9,5,4 (odd TX: the TMA path honours it): tile seams at box index 2 + 8 b (i), 2 + 4 b (j), k chunks from
    2 + 4 b.  The jump is placed on the seam face and one cell past it; the variable is read at every launch."""
    tx, ty, kc = 9, 5, 4
    at = {"contact_i": 2 + (tx - 1), "contact_j": 2 + (ty - 1), "contact_k": 2 + kc}.get(regime)
    at = None if at is None else at + seam
    prm, hb = R.regime_case(regime, SHAPE, at=at)
    assert_reaches(prm, hb, regime, _sensor_keys(regime, SCALAR))
    ref = oracle_residual(prm, hb, RES_FLOW | RES_TURB)
    old = os.environ.get("ADFB_TILE")
    os.environ["ADFB_TILE"] = "%d,%d,%d" % (tx, ty, kc)
    try:
        dw = _residual(prm, hb, RES_FLOW | RES_TURB | RES_SKIP_PREAMBLE)
    finally:
        if old is None:
            del os.environ["ADFB_TILE"]
        else:
            os.environ["ADFB_TILE"] = old
    _rows_close(hb, regime, dw, ref.dw, range(6), TOL, at=at)


@pytest.mark.parametrize("regime", ["floors", "supersonic", "low_mach"])
def test_residual_with_preamble_in_regimes(cuda_lib, regime):
    """adfb_residual with the state preparation (pressure floor 1e-4 pInfCorr, and whalo2's computeEtotBlock on the owned
    cells from the floored pressure), BCs and the whole core"""
    prm, hb = R.regime_case(regime, SHAPE)
    assert_reaches(prm, hb, regime, {"floors": ["p_floor"], "supersonic": ["ff_sup_in", "ff_sup_out"],
                                     "low_mach": ["ff_sub_in", "ff_sub_out"]}[regime])
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(RES_FLOW | RES_TURB)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.residual(RES_FLOW | RES_TURB)
        dw = s.downloadResidual(0)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    ow = hb.d.owned()
    if regime == "floors":
        assert (ho.p[ow] == R.PRESSURE_FLOOR * prm.pInfCorr).any()
    assert rel_max(p[ow], ho.p[ow]) < 1e-14
    _rows_close(hb, regime, dw, ho.dw, range(6), TOL)


# ---------------------------------------------------------------------------------------------------------------------
# boundary conditions
@pytest.mark.parametrize("regime,eq", [("supersonic", "RANS"), ("supersonic", "Euler"), ("low_mach", "RANS"),
                                       ("low_mach", "Euler"), ("contact_k", "RANS")])
def test_bcs_in_regimes(cuda_lib, regime, eq):
    prm, hb = R.regime_case(regime, SHAPE, {"equationType": eq})
    if regime != "contact_k":
        assert_reaches(prm, hb, regime, ["ff_sub_in", "ff_sub_out"] + (["ff_sup_in", "ff_sup_out"] if regime == "supersonic" else []))
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True)
    o.apply_flow_bc(True)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    assert np.abs(w - hb.w).max() > 0
    for name, a, b in (("w", w, ho.w), ("p", p, ho.p), ("rlv", rlv, ho.rlv), ("rev", rev, ho.rev)):
        assert np.isfinite(a).all(), name
        assert rel_max(a, b) < 1e-13, "%s: rel max %.3e" % (name, rel_max(a, b))


# ---------------------------------------------------------------------------------------------------------------------
# smoothers
def _smoother_start(prm, hb):
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(prm.cdisRK[0])
    return ho, o


@pytest.mark.parametrize("regime", ["contact_pocket", "supersonic", "low_mach", "stagnation", "low_reynolds"])
@pytest.mark.parametrize("avg", ["never", "alternate"])
def test_rk_cycle_in_regimes(cuda_lib, regime, avg):
    """contact_pocket, not a block-spanning contact: the latter diverges within one explicit cycle in the reference's
    executeRkStage as in the oracle (tests/regimes.py)"""
    prm, hb = R.regime_case(regime, (16, 12, 10), {"nRKStages": 5, "resAveraging": avg})
    assert_reaches(prm, hb, regime, {"contact_pocket": ["sensor_cap_i", "sensor_cap_j", "sensor_cap_k"],
                                     "supersonic": ["sensor_cap_i", "ff_sup_in", "ff_sup_out"], "low_mach": ["ff_sub_in"],
                                     "stagnation": ["stagnant_j"], "low_reynolds": ["low_cell_re"]}[regime])
    ho, o = _smoother_start(prm, hb)
    dw0 = ho.dw.copy()
    o.rk_smoother()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        dw_dev0 = s.downloadResidual(0)
        s.rkCycle()
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    _rows_close(hb, regime, dw_dev0, dw0, range(5), TOL, what="dw before the cycle")
    ow = hb.d.owned()
    dwv, dwo = w[ow] - hb.w[ow], ho.w[ow] - hb.w[ow]
    assert np.isfinite(ho.w).all() and np.abs(dwo[..., :5]).max() > 1e-8
    for l in range(5):
        assert rel_l2(dwv[..., l], dwo[..., l]) < 1e-10, ("state change", l, rel_l2(dwv[..., l], dwo[..., l]))
    assert rel_max(p, ho.p) < 1e-11


@pytest.mark.parametrize("regime,eq", [("contact_pocket", "RANS"), ("supersonic", "RANS"), ("supersonic", "Euler"),
                                       ("stagnation", "RANS"), ("low_reynolds", "RANS"), ("low_reynolds", "laminar NS")])
def test_dadi_step_in_regimes(cuda_lib, regime, eq):
    prm, hb = R.regime_case(regime, (14, 11, 9), {"equationType": eq})
    assert_reaches(prm, hb, regime, {"supersonic": ["supersonic_i"], "stagnation": ["stagnant_j"],
                                     "low_reynolds": ["low_cell_re"]}.get(regime, ["sensor_cap_i", "sensor_cap_k"]))
    ho, o = _smoother_start(prm, hb)
    o.dadi_step()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        s.dadiStep()
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-10, ("dw after DADI", l, rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]))
        dv, do = w[ow + (l,)] - hb.w[ow + (l,)], ho.w[ow + (l,)] - hb.w[ow + (l,)]
        assert rel_l2(dv, do) < 1e-9, ("state change", l, rel_l2(dv, do))
    assert rel_max(p, ho.p) < 1e-11


def _sa_solve_matches(prm, hb0, niter=1):
    ho = hb0.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    for _ in range(niter):
        o.sa_block()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb0)
        s.applyBCs(True, True)
        s.turbSolveDDADI(niter)
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb0.d.owned()
    assert rel_l2(dw[ow + (5,)], ho.dw[ow + (5,)]) < 1e-10
    dn, do = w[ow + (5,)] - hb0.w[ow + (5,)], ho.w[ow + (5,)] - hb0.w[ow + (5,)]
    assert np.abs(do).max() > 0
    assert rel_l2(dn, do) < 1e-9, rel_l2(dn, do)
    assert rel_max(w[..., 5], ho.w[..., 5]) < 1e-10
    d = hb0.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    assert rel_max(rev[c1], ho.rev[c1]) < 1e-10


@pytest.mark.parametrize("regime", ["stagnation", "supersonic", "contact_k", "low_reynolds"])
def test_sa_ddadi_in_regimes(cuda_lib, regime):
    prm, hb = R.regime_case(regime, SHAPE)
    assert_reaches(prm, hb, regime, {"stagnation": ["sa_rr_clip"], "supersonic": ["ff_sup_in"],
                                     "low_reynolds": ["low_cell_re"]}.get(regime, ["sensor_cap_k"]))
    _sa_solve_matches(prm, hb, 2)


# ---------------------------------------------------------------------------------------------------------------------
# Newton-Krylov products
def _state_vec(hb):
    return np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()


def test_form_function_and_mffd_with_setw_clip_and_pressure_floor(cuda_lib):
    prm, hb = R.regime_case("floors", SHAPE)
    assert_reaches(prm, hb, "floors", ["p_floor", "turb_clip"])
    U = _state_vec(hb)
    assert (U[5::6] < R.TURB_CLIP * prm.wInf[5]).any()
    ref = oracle_form_function(prm, hb, U)
    a = np.random.default_rng(5).standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-7
    ref1 = oracle_form_function(prm, hb, U + h * a)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        r = s.formFunction(U)
        s.mffdSetBase(U)
        y = s.mffdApply(a, h)
    finally:
        s.close()
    assert np.isfinite(r).all()
    assert rel_l2(r, ref) < TOL, rel_l2(r, ref)
    # the product differences two residuals that each agree to ~1e-12 with the oracle's: agreement ~1e-12 |F| / (h |J a|)
    yref = (ref1 - ref) / h
    assert rel_l2(y, yref) < 1e-4, rel_l2(y, yref)


# ---------------------------------------------------------------------------------------------------------------------
# line solves at the lengths where the dispatch changes kernel
@pytest.mark.parametrize("shape", [(129, 17, 16), (97, 15, 16), (128, 16, 15), (96, 97, 9), (256, 9, 8)])
def test_sa_line_solve_lengths(cuda_lib, shape):
    """k_sa_thomas (< 16 cells), k_sa_thomas_part<8,12> (16-96), <8,16> (97-128), <16,16> (129-256): every line length
    of these blocks sits on one side of a boundary 15/16, 96/97, 128/129, 256"""
    from util import case

    prm, hb = case(*shape)
    _sa_solve_matches(prm, hb, 1)


@pytest.mark.parametrize("shape", [(8, 4, 8), (9, 3, 11), (33, 8, 4), (8, 33, 9)])
def test_dadi_line_counts_and_lengths(cuda_lib, shape):
    """k_dadi_thomas_tile runs one warp per 32 lines and splits lines into chunks of 8: 32 / 33 i lines, lengths 8 / 9"""
    from util import case

    prm, hb = case(*shape)
    ho, o = _smoother_start(prm, hb)
    o.dadi_step()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        s.dadiStep()
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        dv, do = w[ow + (l,)] - hb.w[ow + (l,)], ho.w[ow + (l,)] - hb.w[ow + (l,)]
        assert rel_l2(dv, do) < 1e-9, ("state change", l, rel_l2(dv, do))
    assert rel_max(p, ho.p) < 1e-11


# ---------------------------------------------------------------------------------------------------------------------
# low Reynolds number: free-stream pressure 2 Pa (tests/regimes.py), where the viscous flux, the heat flux and the SA
# source terms are 1e-2 .. 1 of the rows they enter (tests/test_low_reynolds_terms.py) instead of 1e-6 .. 1e-4, so
# that the tolerances of this file hold each of those terms to 1e-10 .. 1e-11 of its own size.
LOW_RE = "low_reynolds"
ISO_EXTRAP_FACES = {1: 5, 2: 3, 3: 1, 4: 3, 5: 6, 6: 5}  # iMin extrap, jMin symm, kMin isothermal wall, kMax extrap


def _low_re(shape, options=None, **kw):
    prm, hb = R.regime_case(LOW_RE, shape, options, **kw)
    assert_reaches(prm, hb, LOW_RE)
    return prm, hb


@pytest.mark.parametrize("options,flags", [
    ({"useQCR": True}, 0), ({"useft2SA": False}, 0), ({"turbulenceProduction": "vorticity"}, 0),
    ({"turbulenceOrder": "second order"}, 0), ({"equationType": "laminar NS", "discretization": MATRIX}, 0),
    ({"equationType": "laminar NS", "discretization": UPWIND}, 0),
    ({}, RES_DISS_APPROX | RES_VISC_APPROX), ({"equationType": "laminar NS"}, RES_DISS_APPROX | RES_VISC_APPROX),
    ({"discretization": MATRIX}, RES_DISS_APPROX | RES_VISC_APPROX)])
def test_residual_at_low_reynolds(cuda_lib, options, flags):
    """dw, dtl and the radii of adfb_residual against the oracle; DISS_APPROX | VISC_APPROX selects the thin-layer
    viscousFluxApprox"""
    from test_residual_parity import compare

    prm, hb = _low_re(SHAPE, options)
    if flags & RES_DISS_APPROX:   # the approximate dissipation reads the frozen shock sensor, in hb for the oracle
        Oracle(hb, prm).reference_shock_sensor()
        assert np.abs(hb.shock).max() > 0
    compare(prm, hb, RES_FLOW | (RES_TURB if prm.equations == 3 else 0) | flags)


@pytest.mark.parametrize("shape,tile", [(SHAPE, "9,5,4"), ((20, 14, 9), None), ((40, 24, 16), None)])
@pytest.mark.parametrize("eq", ["RANS", "laminar NS"])
def test_residual_at_low_reynolds_across_tile_seams(cuda_lib, shape, tile, eq):
    """ADFB_TILE=9,5,4 on the default shape, and the tiles the host picks for two larger blocks (5 x 4 and 7 x 13
    cells with k chunks of 2 on 132 SMs): the nodal gradients of the tile kernel live in shared memory and feed the
    viscous flux only, which here is large enough that a gradient wrong at a tile or k-chunk seam fails the row"""
    prm, hb = _low_re(shape, {"equationType": eq})
    flags = RES_FLOW | (RES_TURB if eq == "RANS" else 0)
    ref = oracle_residual(prm, hb, flags)
    old = os.environ.get("ADFB_TILE")
    if tile is not None:
        os.environ["ADFB_TILE"] = tile
    try:
        dw = _residual(prm, hb, flags | RES_SKIP_PREAMBLE)
    finally:
        if old is None:
            os.environ.pop("ADFB_TILE", None)
        else:
            os.environ["ADFB_TILE"] = old
    _rows_close(hb, LOW_RE, dw, ref.dw, range(hb.nw if eq == "RANS" else 5), TOL)


@pytest.mark.parametrize("eq", ["RANS", "laminar NS"])
def test_residual_with_preamble_at_low_reynolds(cuda_lib, eq):
    """adfb_residual with the state preparation (Sutherland rlv, saEddyViscosity) and the BCs on the device, on the
    isothermal-wall layout, whose wall heat flux is a few per cent of the energy row here"""
    prm, hb = _low_re(SHAPE, {"equationType": eq}, physical_faces=ISO_EXTRAP_FACES)
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = hb.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm), 2, d.il, 2, d.jl, 2, d.kl)
    flags = RES_FLOW | (RES_TURB if eq == "RANS" else 0)
    o.residual_core(flags)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.residual(flags)
        dw = s.downloadResidual(0)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    ow = hb.d.owned()
    assert rel_max(rlv[ow], ho.rlv[ow]) < 1e-14
    if eq == "RANS":
        assert rel_max(rev[ow], ho.rev[ow]) < 1e-13
    _rows_close(hb, LOW_RE, dw, ho.dw, range(hb.nw), TOL)


@pytest.mark.parametrize("eq", ["RANS", "laminar NS"])
def test_smoother_residual_and_time_step_at_low_reynolds(cuda_lib, eq):
    """adfb_timestep (dtl with its viscous part, directionally scaled radii) and adfb_smoother_residual at the three
    dissipative stages of the 5-stage scheme, rFil = cdisRK 1.0, 0.56, 0.44: dw and the persistent fw (dissipative and
    viscous part, blended from stage to stage) each against the oracle's residual_block"""
    prm, hb = _low_re(SHAPE, {"equationType": eq, "nRKStages": 5})
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    stages = [st for st in range(5) if prm.cdisRK[st] != 0.0]
    assert [prm.cdisRK[st] for st in stages] == [1.0, 0.56, 0.44]
    ref = []
    for st in stages:
        o.residual_block(prm.cdisRK[st])
        ref.append((ho.dw.copy(), ho.fw.copy()))
    s = ADFLOW_B200(prm)
    got = []
    try:
        s.addBlock(hb)
        s.applyBCs(True, True)
        s.timeStep(False)
        inter = s.downloadIntermed(0)
        for st in stages:
            s.smootherResidual(st)
            got.append((s.downloadResidual(0), s.downloadArray(0, "fw", 5)))
    finally:
        s.close()
    d = hb.d
    ow = d.owned()
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    for n in ("radI", "radJ", "radK"):
        assert rel_max(inter[n], getattr(ho, n)[c1]) < TOL, n
    assert rel_max(inter["dtl"][1:-1, 1:-1, 1:-1], ho.dtl[ow]) < TOL
    for st, (dw, fw), (dwo, fwo) in zip(stages, got, ref):
        _rows_close(hb, LOW_RE, dw, dwo, range(5), TOL, what="dw at stage %d" % st)
        _rows_close(hb, LOW_RE, fw, fwo, range(5), TOL, what="fw at stage %d" % st)


@pytest.mark.parametrize("eq", ["RANS", "laminar NS"])
def test_form_function_and_mffd_at_low_reynolds(cuda_lib, eq):
    """adfb_form_function one-shot and as a slab pipeline (page-locked vectors, ADFB_FF_PIPE), and the product with a
    fixed h"""
    import torch

    prm, hb = _low_re((16, 12, 24), {"equationType": eq})
    U = _state_vec(hb)
    U = U * (1.0 + 1e-3 * np.random.default_rng(3).standard_normal(U.size))
    ref = oracle_form_function(prm, hb, U)
    a = np.random.default_rng(5).standard_normal(U.size) * np.abs(U).clip(1e-6)
    h = 1e-7
    ref1 = oracle_form_function(prm, hb, U + h * a)
    s = ADFLOW_B200(prm)
    old = os.environ.get("ADFB_FF_PIPE")
    try:
        s.addBlock(hb)
        r = s.formFunction(U)
        n = s.getStateSize()
        hw, hr = (torch.empty(n, dtype=torch.float64).pin_memory() for _ in range(2))
        hw.numpy()[:] = U
        hr.numpy()[:] = np.nan
        os.environ["ADFB_FF_PIPE"] = "4"
        s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        r_pipe = hr.numpy().copy()
        s.mffdSetBase(U)
        y = s.mffdApply(a, h)
    finally:
        if old is None:
            os.environ.pop("ADFB_FF_PIPE", None)
        else:
            os.environ["ADFB_FF_PIPE"] = old
        s.close()
    assert np.isfinite(r).all() and np.isfinite(r_pipe).all()
    assert rel_l2(r, ref) < TOL, rel_l2(r, ref)
    assert rel_l2(r_pipe, ref) < 1e-11, rel_l2(r_pipe, ref)
    # the product differences two residuals that each agree to ~1e-12 with the oracle's: agreement ~1e-12 |F| / (h |J a|)
    yref = (ref1 - ref) / h
    assert rel_l2(y, yref) < 1e-4, rel_l2(y, yref)


@pytest.mark.parametrize("coupled,fullvisc", [(False, False), (True, False), (True, True)])
def test_ank_operator_at_low_reynolds(cuda_lib, coupled, fullvisc):
    """adfb_ank_time_step_mat (reads dtl, whose viscous part is large here) and adfb_ank_form_function; useFullVisc
    off selects the thin-layer viscous flux"""
    from adflow_b200.params import make_ank_params
    from test_ank_gpu import oracle_ank_function, oracle_blocks, vec_of

    prm, hb = _low_re((11, 9, 8))
    ank = make_ank_params(cfl=5.0, coupled=coupled, mach=0.8, cflLimit=50.0, turbCFLScale=2.0, useFullVisc=fullvisc)
    ns = hb.nw if coupled else 5
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    o.call("orc_speed_of_sound", C.byref(prm))
    o.reference_shock_sensor()
    T = oracle_blocks(prm, ank, hb)
    U = vec_of(hb, ns)
    v = U * (1.0 + 0.01 * np.random.default_rng(5).standard_normal(U.size))
    Fref = oracle_ank_function(prm, ank, hb, T, v)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.ankSetParams(ank)
        s.referenceShockSensor()
        s.residual(RES_FLOW | RES_TURB | 4)        # useUpdateIntermed: dtl, spectral radii (and aa) of the current state
        s.ankTimeStepMat()
        F = s.ankFormFunction(v)
    finally:
        s.close()
    assert np.abs(np.einsum("qlm,qm->ql", T, v.reshape(-1, ns))).max() > 0
    assert rel_l2(F, Fref) < 1e-11, rel_l2(F, Fref)


def test_mg_3w_cycle_at_low_reynolds(cuda_lib):
    """one 3W cycle on a RANS block: coarse levels with frozen rev and first-order dissipation"""
    from adflow_b200 import synthetic as syn
    from test_mg_gpu import device, oracle_mg_cycle, prepare_fine

    prm, fine = _low_re((16, 16, 8))
    Oracle(fine, prm).apply_turb_bc(True)
    Oracle(fine, prm).apply_flow_bc(True)
    levels = [fine]
    for _ in range(2):
        levels.append(syn.make_coarse_block(levels[-1], prm))
    dev_levels = [l.copy() for l in levels]
    cyc = ADFLOW_B200.cycleStrategy("3w")
    prepare_fine(Oracle(levels[0], prm))
    w0 = levels[0].w.copy()
    oracle_mg_cycle(prm, levels, cyc)
    s = device(prm, dev_levels)
    try:
        s.timeStep(False)
        s.smootherResidual(0)
        s.mgCycle(cyc)
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = fine.d.owned()
    for l in range(5):
        a, b = w[ow + (l,)] - w0[ow + (l,)], fine.w[ow + (l,)] - w0[ow + (l,)]
        assert np.isfinite(a).all() and np.abs(b).max() > 0
        assert rel_l2(a, b) < 1e-8, ("state change over the cycle", l, rel_l2(a, b))
        assert rel_l2(dw[ow + (l,)], fine.dw[ow + (l,)]) < 1e-8, ("residual after the cycle", l)
    assert rel_max(w[..., :5], fine.w[..., :5]) < 1e-10
