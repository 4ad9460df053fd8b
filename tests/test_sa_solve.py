"""Spalart-Allmaras DD-ADI solve (a13): oracle self-checks on CPU, device parity on GPU."""
import numpy as np
import pytest

from adflow_b200 import make_params
from adflow_b200 import synthetic as syn
from adflow_b200.solver import ADFLOW_B200
from oracle.pyoracle import Oracle

from util import MANY, case, rel_l2, rel_max


def test_oracle_strong_relaxation_limit():
    """alfaTurb -> 0 makes the scaled diagonal dominate: the three sweeps reduce to
    delta = dvt / (factor*qq) (checks the qq re-multiplication between sweeps, sa.F90:996-998)."""
    prm = make_params()
    prm.alfaTurb = 1e-7
    hb = syn.make_block(10, 9, 8, prm)
    o = Oracle(hb, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    ow = hb.d.owned()
    o.sa_block()
    dvt0 = -hb.dw[ow + (5,)] / hb.volRef[ow]
    qq = hb.scratch[ow + (1,)]
    delta = hb.scratch[ow + (0,)]
    assert np.abs(delta - dvt0 / qq).max() < 1e-6 * np.abs(delta).max()


def test_oracle_sa_residual_row_equals_blockette_row():
    """dw(itu1) written by the block-path sa_block equals the blockette SA row (same formulas
    except the eps clip of the strain production, which is inactive here)."""
    prm, hb = case(12, 10, 8)
    h2 = hb.copy()
    Oracle(hb, prm).residual_core(16)
    o = Oracle(h2, prm)
    o.sa_block()
    ow = hb.d.owned()
    assert rel_l2(h2.dw[ow + (5,)], hb.dw[ow + (5,)]) < 1e-14


@pytest.mark.gpu
@pytest.mark.parametrize("options,shape,niter", [
    (None, (14, 11, 9), 1),
    (None, (9, 12, 7), 3),
    ({"turbulenceOrder": "second order"}, (10, 9, 8), 2),
    ({"turbulenceProduction": "vorticity", "useft2SA": False}, (8, 9, 10), 1),
    (None, (20, 17, 16), 2),      # lines >= 16 cells: partitioned Thomas kernels (8 lanes per line)
    (None, (33, 40, 18), 1),
    pytest.param(None, ((14, 11, 9), MANY), 1, id="MANY"),   # 14 subfaces: the SA wall terms in two launches
])
def test_sa_ddadi_matches_oracle(cuda_lib, options, shape, niter):
    shape, split = shape if len(shape) == 2 else (shape, None)
    prm, hb0 = case(*shape, options, split=split)
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
    dn = w[ow + (5,)] - hb0.w[ow + (5,)]
    do = ho.w[ow + (5,)] - hb0.w[ow + (5,)]
    assert np.abs(do).max() > 0
    assert rel_l2(dn, do) < 1e-9, rel_l2(dn, do)
    assert rel_max(w[..., 5], ho.w[..., 5]) < 1e-10   # halos included (turbulence BCs)
    d = hb0.d
    c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
    assert rel_max(rev[c1], ho.rev[c1]) < 1e-10
