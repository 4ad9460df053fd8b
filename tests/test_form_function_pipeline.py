"""adfb_form_function as a slab pipeline (page-locked host vectors, blocks without exchange partners): host-to-device copy,
kernels and device-to-host copy of ONE call overlap, plane range by plane range.  Same kernels on the same operands as the
one-shot path, so the two must agree to the last bit wherever the tile kernel cuts its k chunks at the same planes, and
to rounding (1e-13) elsewhere (a chunk boundary recomputes a k face with the kernel's prologue code); both are held against the
oracle's FormFunction_mf as well."""
import os

import numpy as np
import pytest

from adflow_b200.solver import ADFLOW_B200

from sa_configs import assert_sa_planes
from util import MANY, MIXED, case, oracle_form_function, rel_l2

pytestmark = pytest.mark.gpu


def state_vec(hb):
    return np.transpose(hb.w[hb.d.owned()], (2, 1, 0, 3)).reshape(-1).copy()


def pinned(n):
    import torch

    return torch.empty(n, dtype=torch.float64).pin_memory()


@pytest.mark.parametrize("shape,options,slabs", [
    ((24, 16, 32), None, 6),
    ((24, 16, 32), None, 3),
    ((17, 13, 30), None, 8),                       # nz not a multiple of the chunk, odd NI (cp.async tiles instead of TMA)
    ((20, 12, 18), {"equationType": "Euler"}, 6),   # no SA row
    ((16, 12, 24), {"equationType": "laminar NS"}, 4),
    # faces split into pieces, piece boundaries along k inside slabs (tests/util.py: split_faces)
    pytest.param(((24, 16, 32), MIXED), None, 6, id="MIXED"),
    pytest.param(((24, 16, 32), MANY), None, 6, id="MANY"),
])
def test_pipelined_form_function(cuda_lib, shape, options, slabs):
    shape, split = shape if len(shape) == 2 else (shape, None)
    prm, hb = case(*shape, options, split=split)
    U = state_vec(hb)
    U = U * (1.0 + 1e-3 * np.random.default_rng(3).standard_normal(U.size))
    r_orc = oracle_form_function(prm, hb, U)
    s = ADFLOW_B200(prm)
    old = os.environ.get("ADFB_FF_PIPE")
    try:
        s.addBlock(hb)
        n = s.getStateSize()
        hw, hr = pinned(n), pinned(n)
        hw.numpy()[:] = U
        os.environ["ADFB_FF_PIPE"] = "0"
        s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        r_one = hr.numpy().copy()
        hr.numpy()[:] = np.nan
        os.environ["ADFB_FF_PIPE"] = str(slabs)
        s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        r_pipe = hr.numpy().copy()
        # a second call (streams and events reused) and a pageable vector (falls back to the one-shot path)
        hr.numpy()[:] = np.nan
        s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n)
        r_pipe2 = hr.numpy().copy()
        r_page = s.formFunction(U)
    finally:
        if old is None:
            os.environ.pop("ADFB_FF_PIPE", None)
        else:
            os.environ["ADFB_FF_PIPE"] = old
        s.close()
    assert np.isfinite(r_pipe).all() and np.abs(r_pipe).max() > 0
    assert np.array_equal(r_pipe, r_pipe2)
    assert np.array_equal(r_page, r_one)
    scale = np.abs(r_one).max()
    assert np.abs(r_pipe - r_one).max() <= 1e-13 * scale, np.abs(r_pipe - r_one).max() / scale
    assert rel_l2(r_pipe, r_orc) < 1e-11
    assert rel_l2(r_one, r_orc) < 1e-11
    # row by row, and the SA row plane by plane: measured with the oracle on the 24 x 16 x 32 block, the SA row is 2.6e-4
    # of the vector's norm, so the whole-vector check lets an error of 7e-8 .. 3e-5 of one SA plane's own norm through
    d = hb.d
    for r, what in ((r_pipe, "pipelined"), (r_one, "one-shot")):
        got, want = (np.transpose(x.reshape(d.nz, d.ny, d.nx, hb.nw), (2, 1, 0, 3)) for x in (r, r_orc))
        for l in range(hb.nw):
            assert rel_l2(got[..., l], want[..., l]) < 1e-11, "%s row %d: rel L2 %.3e" % (what, l, rel_l2(got[..., l], want[..., l]))
        if hb.nw > 5:
            assert_sa_planes(got[..., 5], want[..., 5], l2_tol=1e-11, what=what + " SA row")
