"""The low_reynolds regime (tests/regimes.py, free-stream pressure 2 Pa) makes the viscous, heat-flux and SA terms a
sizeable part of the rows they enter, so that the residual and smoother tolerances bound each term's own error.

A parity test holds a whole row of dw to 1e-12 relative L2; that bounds a term's error only in proportion to its share
of the row.  The share of a term is measured with the oracle as ||dw(full) - dw(term removed)|| / ||dw(full)|| per
row: the viscous flux removed with rlv = rev = 0, the heat flux with Prandtl numbers of 1e300, an SA term by zeroing
its constant on a copy of AdfbParams, QCR by switching it off.  At 20 kPa (every other synthetic case) the laminar
viscous flux is 1.6e-6 .. 5.5e-6 of its rows and the SA destruction 1.7e-5 of the SA row; at 2 Pa each is at least
1e-2, so a 1e-12 row tolerance holds each term to 1e-10 of its own size.  Runs without a GPU and without the
reference."""
import ctypes as C

import numpy as np
import pytest

import regimes as R
from adflow_b200.params import AdfbParams, RANS
from oracle.pyoracle import Oracle
from util import FLOW, TURB, oracle_residual

SHAPE = (14, 11, 10)
FLOOR = 1e-2
RES_TOL = 1e-12            # the residual tolerance of the parity files
MX, MY, MZ, RHOE, NUT = 1, 2, 3, 4, 5
CONFIGS = [("laminar NS", {}), ("RANS", {}), ("RANS", {"useQCR": True}), ("RANS", {"useft2SA": False}),
           ("RANS", {"turbulenceProduction": "vorticity"}), ("RANS", {"turbulenceOrder": "second order"})]
IDS = ["laminar", "RANS", "QCR", "noft2", "vorticity", "turb2nd"]
# QCR adds to the stress a term in the products of vorticity and strain.  Its share of the momentum rows is that term
# against the whole viscous stress and the inviscid flux, and of the energy row the work of that term against the
# work of the whole stress and the heat flux; once the viscous terms dominate, lowering the pressure does not raise
# either.  Measured on this block: mx 1.8e-3, my 1.2e-3, mz 4.8e-2, rhoE 6.4e-5 at 2 Pa; 3.2e-3, 1.1e-2, 0.40, 6.4e-5
# at 0.2 Pa; 2.3e-7, 1.2e-7, 4.8e-6, 8.7e-8 at 20 kPa.  The floors below are those of 2 Pa with a margin of 2.
QCR_FLOORS = {MX: 8e-4, MY: 6e-4, MZ: FLOOR, RHOE: 3e-5}


def _copy(prm):
    p = AdfbParams()
    C.pointer(p)[0] = prm
    p._muInf = prm._muInf
    return p


def _share(full, removed, ow, l):
    a, b = full[ow + (l,)], removed[ow + (l,)]
    assert np.isfinite(b).all(), l
    return np.linalg.norm((a - b).ravel()) / np.linalg.norm(a.ravel())


def _flags(prm):
    return FLOW | TURB if prm.equations == RANS else FLOW


def _case(eq, options):
    prm, hb = R.regime_case("low_reynolds", SHAPE, dict(options, equationType=eq))
    return prm, hb, oracle_residual(prm, hb, _flags(prm))


def _assert_shares(what, full, removed, ow, floors):
    shares = {l: _share(full, removed, ow, l) for l in floors}
    low = {l: "%.2e" % s for l, s in shares.items() if not s >= floors[l]}
    assert not low, "%s: shares %s below the floors %s" % (what, low, floors)


@pytest.mark.parametrize("eq,options", CONFIGS, ids=IDS)
def test_viscous_and_heat_flux_are_visible(eq, options):
    prm, hb, full = _case(eq, options)
    ow = hb.d.owned()
    h0 = hb.copy()
    h0.rlv[...] = 0.0
    h0.rev[...] = 0.0
    _assert_shares("viscous flux", full.dw, oracle_residual(prm, h0, FLOW).dw, ow, dict.fromkeys((MX, MY, MZ, RHOE), FLOOR))
    p = _copy(prm)
    p.prandtl = p.prandtlTurb = 1e300
    _assert_shares("heat flux", full.dw, oracle_residual(p, hb, _flags(prm)).dw, ow, {RHOE: FLOOR})
    if prm.useQCR:
        p = _copy(prm)
        p.useQCR = 0
        _assert_shares("QCR", full.dw, oracle_residual(p, hb, _flags(prm)).dw, ow, QCR_FLOORS)


@pytest.mark.parametrize("eq,options", CONFIGS[1:], ids=IDS[1:])
@pytest.mark.parametrize("const", ["rsaCw1", "rsaCb2"])
def test_sa_destruction_and_cross_diffusion_are_visible(eq, options, const):
    prm, hb, full = _case(eq, options)
    p = _copy(prm)
    setattr(p, const, 0.0)
    _assert_shares(const, full.dw, oracle_residual(p, hb, _flags(prm)).dw, hb.d.owned(), {NUT: FLOOR})


@pytest.mark.parametrize("eq,options", CONFIGS, ids=IDS)
def test_a_1e_9_viscosity_error_fails_the_residual_tolerance(eq, options):
    """rlv and rev x (1 + 1e-9), which is what a float intermediate or a slightly wrong constant in the viscous flux
    does: every row the viscosities enter moves by more than 10x the residual tolerance"""
    prm, hb, full = _case(eq, options)
    h1 = hb.copy()
    h1.rlv *= 1.0 + 1e-9
    h1.rev *= 1.0 + 1e-9
    rows = (MX, MY, MZ, RHOE) + ((NUT,) if prm.equations == RANS else ())
    _assert_shares("rlv, rev x (1 + 1e-9)", full.dw, oracle_residual(prm, h1, _flags(prm)).dw, hb.d.owned(),
                   dict.fromkeys(rows, 10 * RES_TOL))


@pytest.mark.parametrize("eq", ["laminar NS", "RANS"])
def test_viscous_parts_of_the_smoother_residual_and_time_step_are_visible(eq):
    """residual_block's fw (dissipative plus viscous part, rFil 1) and the viscous part of dtl, max over cells"""
    prm, hb = R.regime_case("low_reynolds", SHAPE, {"equationType": eq})
    out = []
    for visc in (True, False):
        h = hb.copy()
        if not visc:
            h.rlv[...] = 0.0
            h.rev[...] = 0.0
        o = Oracle(h, prm)
        o.time_step(True)
        h.fw[...] = 0.0
        o.residual_block(1.0)
        out.append(h)
    ow = hb.d.owned()
    _assert_shares("viscous part of fw", out[0].fw, out[1].fw, ow, dict.fromkeys((MX, MY, MZ, RHOE), FLOOR))
    inv_full, inv_inviscid = 1.0 / out[0].dtl[ow], 1.0 / out[1].dtl[ow]
    assert (np.abs(inv_full - inv_inviscid) / inv_full).max() > FLOOR


def test_the_terms_are_invisible_at_20_kpa():
    """the reason for the regime: the default free-stream pressure leaves the laminar viscous flux below 1e-5 of its
    rows and the SA destruction below 1e-4 of the SA row"""
    from util import case

    for eq in ("laminar NS", "RANS"):
        prm, hb = case(*SHAPE, {"equationType": eq})
        full = oracle_residual(prm, hb, _flags(prm))
        ow = hb.d.owned()
        if eq == "laminar NS":
            h0 = hb.copy()
            h0.rlv[...] = 0.0
            removed = oracle_residual(prm, h0, FLOW)
            assert max(_share(full.dw, removed.dw, ow, l) for l in (MX, MY, MZ, RHOE)) < 1e-5
        else:
            p = _copy(prm)
            p.rsaCw1 = 0.0
            assert _share(full.dw, oracle_residual(p, hb, FLOW | TURB).dw, ow, NUT) < 1e-4
