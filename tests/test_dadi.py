"""DADI smoother (a15): oracle self-checks on CPU, device parity on GPU."""
import numpy as np
import pytest

from adflow_b200.solver import ADFLOW_B200
from oracle.pyoracle import Oracle

from util import case, rel_l2, rel_max


def prepared(options=None, shape=(14, 11, 9)):
    prm, hb = case(*shape, options)
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    hb.fw[...] = 0
    o.residual_block(1.0)
    return prm, hb


def test_oracle_dadi_reduces_to_explicit_step_for_tiny_cfl():
    """cfl -> 0: the implicit operator tends to the identity, so computedwDADI returns
    -(-cfl*dtl*vol*dw)/vol = cfl*dtl*dw up to O(cfl^2) (changes of basis must cancel)."""
    prm, hb = prepared({"CFL": 1e-6})
    o = Oracle(hb, prm)
    ow = hb.d.owned()
    dw0 = hb.dw.copy()
    d = hb.d
    for l in range(5):
        hb.dw[ow + (l,)] *= -prm.cfl * hb.dtl[ow] * hb.vol[ow]
    o.compute_dw_dadi()
    exp = prm.cfl * hb.dtl[ow][..., None] * dw0[ow + (slice(0, 5),)]
    assert rel_l2(hb.dw[ow + (slice(0, 5),)], exp) < 1e-4


def test_oracle_dadi_smoother_reduces_residual():
    prm, hb = prepared({"equationType": "Euler", "CFL": 2.0})
    o = Oracle(hb, prm)
    n0 = o.norms()[1]
    for _ in range(15):
        o.dadi_step()
        o.time_step(True)
        o.residual_block(1.0)
    assert np.isfinite(hb.w).all()
    assert o.norms()[1] < n0


@pytest.mark.gpu
@pytest.mark.parametrize("options,shape", [
    (None, (14, 11, 9)),
    ({"equationType": "Euler", "CFL": 3.0}, (12, 9, 10)),
    ({"equationType": "laminar NS"}, (9, 12, 8)),
    ({"resAveraging": "always", "CFL": 5.0}, (10, 9, 8)),
    (None, (1, 7, 6)),
    (None, (20, 17, 16)),         # lines >= 16 cells: partitioned Thomas kernels (8 lanes per line)
    ({"resAveraging": "always", "CFL": 5.0}, (33, 18, 40)),
    ({"equationType": "Euler"}, (16, 35, 9)),   # mixed: i, j partitioned, k serial
    ({"discretization": "central plus matrix dissipation", "equationType": "Euler"}, (12, 9, 10)),
    ({"discretization": "upwind", "equationType": "laminar NS"}, (12, 9, 10)),
    ({"discretization": "upwind"}, (12, 9, 10)),
    # line lengths for each lines-per-CTA of the shared-memory solve (ADFB_DADI_SMEM=1, 14 arrays of nl (L + 1) doubles
    # in 220 KiB): L = 32 up to 60 cells, 16 up to 118, 8 up to 223, 4 up to 402
    (None, (60, 61, 4)),
    (None, (118, 119, 3)),
    (None, (223, 224, 2)),
    ({"equationType": "Euler"}, (402, 7, 3)),
])
def test_dadi_step_matches_oracle(cuda_lib, options, shape):
    prm, hb0 = case(*shape, options)
    ho = hb0.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(1.0)
    o.dadi_step()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb0)
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        s.dadiStep()
        w, p, rlv, rev = s.downloadState(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = hb0.d.owned()
    for l in range(5):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-10, ("dw after DADI", l, rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]))
    dwv = w[ow] - hb0.w[ow]
    dwo = ho.w[ow] - hb0.w[ow]
    for l in range(5):
        assert rel_l2(dwv[..., l], dwo[..., l]) < 1e-9, ("state change", l)
    assert rel_max(p, ho.p) < 1e-11
