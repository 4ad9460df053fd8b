"""Approximate (preconditioner / ANK) flux variants (a8): *Approx dissipation with the frozen
shock sensor and the thin-layer viscous flux, selected with the blocketteRes flags."""
import numpy as np
import pytest

from adflow_b200.solver import ADFLOW_B200, RES_DISS_APPROX, RES_FLOW, RES_SKIP_PREAMBLE, RES_TURB, RES_VISC_APPROX
from oracle.pyoracle import Oracle

from util import case, rel_l2, rel_max

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("disc", ["central plus scalar dissipation", "central plus matrix dissipation", "upwind"])
@pytest.mark.parametrize("approx", [RES_DISS_APPROX, RES_VISC_APPROX, RES_DISS_APPROX | RES_VISC_APPROX])
def test_rans_approx_variants(cuda_lib, disc, approx):
    prm, hb = case(13, 10, 9, {"discretization": disc})
    # sensor frozen at a different (earlier) state than the one the residual is evaluated at
    frozen = hb.copy()
    frozen.w[..., 0] *= 1.0 + 0.01 * np.sin(np.arange(frozen.w[..., 0].size)).reshape(frozen.w[..., 0].shape, order="F")
    of = Oracle(frozen, prm)
    of.reference_shock_sensor()
    ho = hb.copy()
    ho.shock[...] = frozen.shock
    flags = RES_FLOW | RES_TURB | approx
    Oracle(ho, prm).residual_core(flags)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(frozen)
        s.referenceShockSensor()
        s.uploadState(0, hb)
        s.residual(flags | RES_SKIP_PREAMBLE)
        dw = s.downloadResidual(0)
        shock = s.downloadArray(0, "shock")
    finally:
        s.close()
    assert rel_max(shock, frozen.shock) < 1e-13
    ow = hb.d.owned()
    for l in range(6):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-11, (l, rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]))
    # the approximate residual really differs from the exact one
    he = hb.copy()
    Oracle(he, prm).residual_core(RES_FLOW | RES_TURB)
    assert rel_l2(ho.dw[ow + (1,)], he.dw[ow + (1,)]) > 1e-6


def euler_approx_case(disc, approx):
    """An inviscid block has no viscous flux, so VISC_APPROX alone leaves the exact residual (blockette.F90:636-644)."""
    prm, hb = case(12, 9, 8, {"equationType": "Euler", "discretization": disc})
    ho = hb.copy()
    o = Oracle(ho, prm)
    o.reference_shock_sensor()
    o.residual_core(RES_FLOW | approx)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.referenceShockSensor()
        s.residual(RES_FLOW | approx | RES_SKIP_PREAMBLE)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-11, (l, rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]))
    he = hb.copy()
    Oracle(he, prm).residual_core(RES_FLOW)
    if approx & RES_DISS_APPROX:   # the approximate dissipation really differs from the exact one
        assert rel_l2(ho.dw[ow + (1,)], he.dw[ow + (1,)]) > 1e-6
    else:
        assert np.array_equal(ho.dw[ow + (slice(0, 5),)], he.dw[ow + (slice(0, 5),)])


def test_euler_diss_approx(cuda_lib):
    euler_approx_case("central plus scalar dissipation", RES_DISS_APPROX)


# every other pair of discretisation and approximate flags (scalar + DISS is test_euler_diss_approx)
EULER_APPROX = [(d, f) for d in ("scalar", "matrix", "upwind") for f in ("DISS", "VISC", "DISS_VISC") if (d, f) != ("scalar", "DISS")]
DISCS = {"scalar": "central plus scalar dissipation", "matrix": "central plus matrix dissipation", "upwind": "upwind"}
FLAGS = {"DISS": RES_DISS_APPROX, "VISC": RES_VISC_APPROX, "DISS_VISC": RES_DISS_APPROX | RES_VISC_APPROX}


@pytest.mark.parametrize("disc,flags", EULER_APPROX, ids=["%s-%s" % c for c in EULER_APPROX])
def test_euler_approx_flags(cuda_lib, disc, flags):
    euler_approx_case(DISCS[disc], FLAGS[flags])
