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
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_SKIP_PREAMBLE, RES_TURB
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
@pytest.mark.parametrize("regime", CONTACTS + ("supersonic", "stagnation"))
@pytest.mark.parametrize("eq,disc", [("RANS", SCALAR), ("laminar NS", SCALAR), ("RANS", MATRIX), ("RANS", UPWIND),
                                     ("Euler", UPWIND)])
def test_residual_in_regimes(cuda_lib, regime, eq, disc):
    if disc == MATRIX and regime in CONTACTS:
        pytest.skip("a contact at constant pressure does not reach the pressure sensor of matrix dissipation")
    prm, hb = R.regime_case(regime, SHAPE, {"equationType": eq, "discretization": disc})
    keys = _sensor_keys(regime, disc) if eq != "Euler" else []
    keys += {"supersonic": ["supersonic_i"], "stagnation": ["stagnant_j"] + (["sa_rr_clip"] if eq == "RANS" else [])}.get(regime, [])
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


@pytest.mark.parametrize("regime", ["contact_pocket", "supersonic", "low_mach", "stagnation"])
@pytest.mark.parametrize("avg", ["never", "alternate"])
def test_rk_cycle_in_regimes(cuda_lib, regime, avg):
    """contact_pocket, not a block-spanning contact: the latter diverges within one explicit cycle in the reference's
    executeRkStage as in the oracle (tests/regimes.py)"""
    prm, hb = R.regime_case(regime, (16, 12, 10), {"nRKStages": 5, "resAveraging": avg})
    assert_reaches(prm, hb, regime, {"contact_pocket": ["sensor_cap_i", "sensor_cap_j", "sensor_cap_k"],
                                     "supersonic": ["sensor_cap_i", "ff_sup_in", "ff_sup_out"], "low_mach": ["ff_sub_in"],
                                     "stagnation": ["stagnant_j"]}[regime])
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
                                       ("stagnation", "RANS")])
def test_dadi_step_in_regimes(cuda_lib, regime, eq):
    prm, hb = R.regime_case(regime, (14, 11, 9), {"equationType": eq})
    assert_reaches(prm, hb, regime, {"supersonic": ["supersonic_i"], "stagnation": ["stagnant_j"]}.get(regime, ["sensor_cap_i", "sensor_cap_k"]))
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


@pytest.mark.parametrize("regime", ["stagnation", "supersonic", "contact_k"])
def test_sa_ddadi_in_regimes(cuda_lib, regime):
    prm, hb = R.regime_case(regime, SHAPE)
    assert_reaches(prm, hb, regime, {"stagnation": ["sa_rr_clip"], "supersonic": ["ff_sup_in"]}.get(regime, ["sensor_cap_k"]))
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
