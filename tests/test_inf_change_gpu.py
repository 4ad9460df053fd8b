"""infChangeCorrection and setUniformFlow on the device (adfb_inf_change_correction, adfb_set_uniform_flow; the Python
layer's infChangeCorrection / setUniformFlow / resetFlow) against the restatement of tests/inf_change.py, which is pinned
bit for bit against the reference's own routines (translated by tests/ref_inf_change.py) in
tests/test_oracle_vs_reference_inf_change.py.

The owned velocities, density and turbulence variable are compared bit for bit.  whalo2 ends with computeEtotBlock on the
owned cells, and the device forms that total energy with FMA contraction (as test_overset_gpu.py notes for the orphan
average), so the owned rho E is held to a few ulp; halos to the 1e-13 of the BC parity tests (test_smoother_parity.py)."""
import numpy as np
import pytest

from adflow_b200 import make_params
from adflow_b200.halo import build_overset_pattern, comm_vars, exchange_numpy, exchange_numpy_overset
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
from oracle.pyoracle import Oracle

import inf_change as IC
from util import MIXED, case, rel_l2, rel_max

pytestmark = pytest.mark.gpu

EQS = ["Euler", "laminar NS", "RANS"]
SHAPE = (13, 11, 9)


def _close(a, b):
    return np.abs(a - b).max() <= 4e-15 * max(1.0, np.abs(b).max())


def _vars(prm):
    return lambda hb: comm_vars(hb, 1, hb.nw, True, True, prm.equations != 1, prm.equations == 3)


def _device(prm, blocks, pattern=None, overset=None):
    s = ADFLOW_B200(prm)
    for hb in blocks:
        s.addBlock(hb)
    if pattern is not None:
        s.setCommPattern(pattern)
    if overset is not None:
        s.setOversetPattern(overset)
    return s


def _states(s, n):
    return [s.downloadState(q) for q in range(n)]


def assert_state(got, hb, exact_owned=True, name=""):
    """got = (w, p, rlv, rev) of the device against the block hb of the restatement"""
    w, p, rlv, rev = got
    ow = hb.d.owned()
    assert np.isfinite(w).all(), name
    for l in range(hb.nw):
        if l == 4 or not exact_owned:
            assert _close(w[ow + (l,)], hb.w[ow + (l,)]), (name, "owned", l)
        else:
            assert np.array_equal(w[ow + (l,)], hb.w[ow + (l,)]), (name, "owned", l, np.abs(w[ow + (l,)] - hb.w[ow + (l,)]).max())
    for a, b, what in ((w, hb.w, "w"), (p, hb.p, "p"), (rlv, hb.rlv, "rlv"), (rev, hb.rev, "rev")):
        assert rel_max(a, b) < 1e-13, (name, what, rel_max(a, b))


def correct_on_device(prm0, prm1, blocks, kind, tol=1e-12, pattern=None, overset=None):
    """state of blocks under prm0, then setParams(prm1) and the correction; returns (applied, states, launches)"""
    s = _device(prm0, blocks, pattern, overset)
    try:
        s.setParams(prm1)
        n0 = s.launchCount()
        applied = s.infChangeCorrection(list(prm0.wInf)[:5], tol, kind)
        s.synchronize()
        return applied, _states(s, len(blocks)), s.launchCount() - n0
    finally:
        s.close()


CHANGES = [("alpha", 2, "offset"), ("alpha", 2, "rotate"), ("alpha", 3, "offset"), ("alpha", 3, "rotate"),
           ("mach", 2, "offset"), ("pressure", 2, "offset"), ("temperature", 2, "offset")]


@pytest.mark.parametrize("layout", ["default", "MIXED"])
@pytest.mark.parametrize("change,lift,kind", CHANGES, ids=["%s-lift%d-%s" % c for c in CHANGES])
@pytest.mark.parametrize("eq", EQS)
def test_correction_matches_restatement(cuda_lib, eq, change, lift, kind, layout):
    prm0, prm1 = IC.free_stream_pair(eq, change, lift)
    hb = case(*SHAPE, IC.options(eq, lift), split=MIXED if layout == "MIXED" else None)[1]
    ref = hb.copy()
    assert IC.inf_change_correction([ref], prm1, list(prm0.wInf)[:5], kind=kind)
    applied, (got,), _ = correct_on_device(prm0, prm1, [hb], kind)
    assert applied
    assert np.abs(got[0] - hb.w).max() > 0
    assert_state(got, ref, name="%s %s %s" % (eq, change, kind))


def row_of_blocks(prm, widths, ny=7, nz=6, seed=314):
    """level-1 blocks of widths[b] x ny x nz cells side by side in i (one mesh, different shapes), and their 1-to-1
    pattern in the layout of adflow_b200.halo.build_cartesian_pattern: same-rank copies only, ordered by receiving
    block, then k, j, i"""
    from adflow_b200 import synthetic as syn

    off = np.concatenate([[0], np.cumsum(widths)])
    nb = len(widths)
    blocks = []
    for b, nx in enumerate(widths):
        faces = [3, 4, 5, 6] + ([1] if b == 0 else []) + ([2] if b == nb - 1 else [])
        blocks.append(syn.make_block(nx, ny, nz, prm, origin=(int(off[b]), 0, 0), global_n=(int(off[-1]), ny, nz), seed=seed,
                                     origin_tag=b, physical_faces=tuple(sorted(faces))))
    donor, halo = [], []
    for rb, nx in enumerate(widths):
        for k in range(2, nz + 2):
            for j in range(2, ny + 2):
                for i in (0, 1, nx + 2, nx + 3):
                    gi = off[rb] + i - 2
                    if gi < 0 or gi >= off[-1]:
                        continue
                    sb = int(np.searchsorted(off, gi, side="right") - 1)
                    donor.append((sb, int(gi - off[sb] + 2), j, k))
                    halo.append((rb, i, j, k))
    i4 = lambda rows: np.array(rows, dtype=np.int32).reshape(-1, 4)  # noqa: E731
    z = np.zeros(0, dtype=np.int32)
    pat = {"nbrRank": z, "sendCount": z, "recvCount": z, "sendList": i4([]), "recvList": i4([]), "donorList": i4(donor),
           "haloList": i4(halo)}
    return blocks, pat


@pytest.mark.parametrize("kind", IC.KINDS)
@pytest.mark.parametrize("eq", EQS)
def test_three_blocks_with_a_one_to_one_pattern(cuda_lib, eq, kind):
    """three level-1 blocks of different shapes exchanging second halos through a 1-to-1 pattern"""
    prm0, prm1 = IC.free_stream_pair(eq, "alpha", 2)
    blocks, pat = row_of_blocks(prm0, (8, 5, 11))
    vars_ = _vars(prm0)
    for hb in blocks:
        Oracle(hb, prm0).apply_flow_bc(True)
    exchange_numpy(blocks, pat, vars_)
    ref = [b.copy() for b in blocks]
    IC.inf_change_correction(ref, prm1, list(prm0.wInf)[:5], kind=kind, exchange=lambda bl: exchange_numpy(bl, pat, vars_))
    applied, got, _ = correct_on_device(prm0, prm1, blocks, kind, pattern=pat)
    assert applied
    for q in range(3):
        assert_state(got[q], ref[q], name="block %d" % q)
    # the exchange moved corrected values into the halos
    unexchanged = [b.copy() for b in blocks]
    IC.inf_change_correction(unexchanged, prm1, list(prm0.wInf)[:5], kind=kind)
    assert np.abs(unexchanged[1].w[0:2] - ref[1].w[0:2]).max() > 0


@pytest.mark.parametrize("eq", EQS)
def test_blocks_of_different_shapes(cuda_lib, eq):
    """three independent level-1 blocks of different shapes in one context"""
    prm0, prm1 = IC.free_stream_pair(eq, "alpha", 3)
    opt = IC.options(eq, 3)
    blocks = [case(*sh, opt, seed=sd)[1] for sh, sd in (((9, 7, 6), 1), ((5, 11, 8), 2), ((12, 6, 10), 3))]
    ref = [b.copy() for b in blocks]
    IC.inf_change_correction(ref, prm1, list(prm0.wInf)[:5], kind="rotate")
    applied, got, _ = correct_on_device(prm0, prm1, blocks, "rotate")
    assert applied
    for q in range(3):
        assert_state(got[q], ref[q], name="block %d" % q)


@pytest.mark.parametrize("kind", IC.KINDS)
def test_overset_pattern_reapplies_the_boundary_conditions(cuda_lib, kind):
    from test_overset_host import overset_entries, two_blocks

    prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
    blocks = two_blocks(prm0)
    pat = build_overset_pattern(overset_entries())
    vars_ = _vars(prm0)
    ref = [b.copy() for b in blocks]
    IC.inf_change_correction(ref, prm1, list(prm0.wInf)[:5], kind=kind,
                             exchange=lambda bl: exchange_numpy_overset(bl, pat, vars_), overset=True)
    applied, got, _ = correct_on_device(prm0, prm1, blocks, kind, overset=pat)
    assert applied
    for q in range(2):
        # the fringe cells of both blocks are owned cells filled by the 8-term interpolation (FMA on the device): a few ulp
        assert_state(got[q], ref[q], exact_owned=False, name="block %d" % q)
    # the re-applied BCs differ from BCs of the exchanged state without them
    no_bc = [b.copy() for b in blocks]
    IC.inf_change_correction(no_bc, prm1, list(prm0.wInf)[:5], kind=kind, exchange=lambda bl: exchange_numpy_overset(bl, pat, vars_))
    assert np.abs(no_bc[1].w - ref[1].w).max() > 0


@pytest.mark.parametrize("case_", ["identical", "lift3-sign-flip", "tol-above"])
def test_skip_launches_nothing_and_keeps_the_state(cuda_lib, case_):
    if case_ == "identical":
        prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
        prm1 = prm0
        tol = 1e-12
    elif case_ == "lift3-sign-flip":
        prm0, prm1 = IC.sign_flip_pair("RANS")
        tol = 1e-12
    else:
        prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
        tol = np.nextafter(IC.my_norm2(IC.delta_winf(prm1, list(prm0.wInf)[:5])), np.inf)
    assert IC.skipped(prm1, list(prm0.wInf)[:5], tol)
    hb = case(*SHAPE, IC.options("RANS", 3 if "lift3" in case_ else 2))[1]
    for kind in IC.KINDS:
        s = _device(prm0, [hb])
        try:
            before = s.downloadState(0)
            s.setParams(prm1)
            s.synchronize()
            n0 = s.launchCount()
            assert not s.infChangeCorrection(list(prm0.wInf)[:5], tol, kind)
            assert s.launchCount() == n0
            after = s.downloadState(0)
        finally:
            s.close()
        for a, b in zip(after, before):
            assert np.array_equal(a, b)


def test_tolerance_just_below_the_change_applies(cuda_lib):
    prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
    tol = IC.my_norm2(IC.delta_winf(prm1, list(prm0.wInf)[:5]))   # norm < tol is false: applied
    hb = case(*SHAPE)[1]
    ref = hb.copy()
    assert IC.inf_change_correction([ref], prm1, list(prm0.wInf)[:5], tol=tol)
    applied, (got,), n = correct_on_device(prm0, prm1, [hb], "offset", tol=tol)
    assert applied and n > 0
    assert_state(got, ref)


def _refused(s, call, nblocks):
    import ctypes as C

    before = _states(s, nblocks)
    with pytest.raises(Exception) as e:
        call()
    buf = C.create_string_buffer(1024)
    s.L.adfb_last_error(buf, 1024)
    assert buf.value, "no message"
    after = _states(s, nblocks)
    for x, y in zip(after, before):
        for a, b in zip(x, y):
            assert np.array_equal(a, b, equal_nan=True)
    return buf.value.decode() + " / " + str(e.value)


def test_refusals(cuda_lib):
    import ctypes as C

    prm0, prm1 = IC.free_stream_pair("RANS", "mach", 2)
    hb = case(*SHAPE)[1]
    old = list(prm0.wInf)[:5]
    s = _device(prm0, [hb])
    try:
        s.setParams(prm1)
        msg = _refused(s, lambda: s.infChangeCorrection(old, 1e-12, "rotate"), 1)   # a change of speed alone
        assert "rotate" in msg
        arr = (C.c_double * 5)(*old)
        flag = C.c_int(7)
        for args in ((arr, 1e-12, 2, C.byref(flag)), (None, 1e-12, 0, C.byref(flag)), (arr, 1e-12, 0, None)):
            rc = [None]

            def call(args=args):
                rc[0] = s.L.adfb_inf_change_correction(*args)
                if rc[0] != 0:
                    raise RuntimeError("refused")
            _refused(s, call, 1)
            assert rc[0] != 0
        with pytest.raises(ValueError):
            s.infChangeCorrection(old, 1e-12, "twist")
    finally:
        s.close()
    # a ground level other than 1
    from adflow_b200 import synthetic as syn

    s = ADFLOW_B200(prm0)
    try:
        s.addBlock(hb)
        s.addCoarseBlock(syn.make_coarse_block(hb, prm0), 0)
        s.setGroundLevel(2)
        s.setParams(prm1)
        assert "ground level" in _refused(s, lambda: s.infChangeCorrection(old, 1e-12, "offset"), 2)
        assert "no block" in _refused(s, lambda: s.setUniformFlow(3, 1e-3, 0.009), 2)
    finally:
        s.close()


def test_refused_without_parameters(cuda_lib):
    """a context whose parameters were never set (adfb_finalize clears them) refuses both entry points"""
    import ctypes as C

    from adflow_b200 import _lib

    L = _lib.load()
    assert L.adfb_init(0, None, 0, 1) == 0
    try:
        arr = (C.c_double * 5)(1.0, 0.5, 0.0, 0.0, 2.5)
        flag = C.c_int(0)
        assert L.adfb_inf_change_correction(arr, 1e-12, 0, C.byref(flag)) != 0
        assert L.adfb_set_uniform_flow(1, 1e-3, 0.009) != 0
        buf = C.create_string_buffer(1024)
        L.adfb_last_error(buf, 1024)
        assert b"adfb_set_params" in buf.value
    finally:
        L.adfb_finalize()


@pytest.mark.parametrize("eq", EQS)
@pytest.mark.parametrize("level", [1, 2])
def test_set_uniform_flow(cuda_lib, eq, level):
    from adflow_b200 import synthetic as syn

    prm, hb = case(12, 10, 8, IC.options(eq, 2))
    coarse = syn.make_coarse_block(hb, prm)
    mu, ratio = 1.7e-3, 0.009
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(hb)
        s.addCoarseBlock(coarse, 0)
        if level == 1:
            s.residual(RES_FLOW | RES_TURB)
            assert np.abs(s.downloadResidual(0)).max() > 0
        before = _states(s, 2)
        s.setUniformFlow(level, mu, ratio)
        got = _states(s, 2)
        dw = [s.downloadResidual(q) for q in range(2)]
        fw = [s.downloadArray(q, "fw", 5) for q in range(2)]
    finally:
        s.close()
    target = hb.copy() if level == 1 else coarse.copy()
    IC.set_uniform_flow(target, prm, mu, ratio)
    q = level - 1
    for a, b in zip(got[q], (target.w, target.p, target.rlv, target.rev)):
        assert np.array_equal(a, b)
    if prm.equations == 1:   # arrays the reference leaves alone stay as they were
        assert np.array_equal(got[q][2], before[q][2]) and np.array_equal(got[q][3], before[q][3])
    assert np.array_equal(dw[q], target.dw) and np.array_equal(fw[q], target.fw)
    for a, b in zip(got[1 - q], before[1 - q]):   # the other level is not touched
        assert np.array_equal(a, b)


@pytest.mark.parametrize("mg_start", [1, 2])
def test_reset_flow_then_full_multigrid_start_up(cuda_lib, mg_start):
    """resetFlow(mgStartLevel) then fullMultigridStartUp against the restatement and the oracle composition of
    tests/fmg_oracle.py (as test_fmg_gpu.py, 1e-9 on the states)"""
    import fmg_oracle as fo
    from test_mg_gpu import device, make_levels

    prm, levels = make_levels((16, 12, 8), {"equationType": "RANS"}, 2)
    mu, ratio = prm._muInf, 0.009
    dev_levels = [hb.copy() for hb in levels]
    IC.set_uniform_flow(levels[mg_start - 1], prm, mu, ratio)
    for hb in levels:
        hb.fw[...] = 0
    snaps = fo.full_multigrid_start_up(prm, levels, mg_start, 2, "2v") if mg_start > 1 else None
    s = device(prm, dev_levels)
    try:
        s.resetFlow(mg_start, mu, ratio)
        assert s.L.adfb_get_ground_level() == mg_start
        s.fullMultigridStartUp(mg_start, 2, "2v")
        if mg_start == 1:   # no coarse ground level to run: the start-up leaves the uniform flow as it is
            assert s.L.adfb_get_ground_level() == 1
            got = s.downloadState(0)
            for a, b in zip(got, (levels[0].w, levels[0].p, levels[0].rlv, levels[0].rev)):
                assert np.array_equal(a, b)
            return
        w, p = s.downloadState(0)[:2]
    finally:
        s.close()
    assert sorted(snaps) == [2]
    assert rel_max(w, levels[0].w) < 1e-9, rel_max(w, levels[0].w)
    assert rel_max(p, levels[0].p) < 1e-9


def _cycle(s):
    s.applyBCs(True, True)
    s.timeStep(False)
    s.smootherResidual(0)
    s.rkCycle()


def _oracle_cycle_change(prm, hb, before):
    ho = hb.copy()
    ho.w[...], ho.p[...], ho.rlv[...], ho.rev[...] = before
    w0 = ho.w.copy()
    o = Oracle(ho, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    o.time_step(True)
    ho.fw[...] = 0
    o.residual_block(prm.cdisRK[0])
    o.rk_smoother()
    return ho.w - w0


@pytest.mark.parametrize("kind", IC.KINDS)
def test_alpha_sweep_on_one_live_context(cuda_lib, kind):
    """RK cycles at alpha 1.8, setParams at alpha 2.8, the correction, more RK cycles: the live context equals a fresh one
    given the corrected state, and every cycle's state change follows the oracle to 1e-10"""
    opt = {"nRKStages": 3, "resAveraging": "never"}
    prm0, hb = case(*SHAPE, opt)
    prm1 = make_params(opt, alpha_deg=2.8)
    ow = hb.d.owned()

    def cycles(s, prm, n):
        for _ in range(n):
            before = s.downloadState(0)
            _cycle(s)
            after = s.downloadState(0)
            ref = _oracle_cycle_change(prm, hb, before)
            for l in range(5):
                a, b = after[0][ow + (l,)] - before[0][ow + (l,)], ref[ow + (l,)]
                assert np.abs(b).max() > 0
                assert rel_l2(a, b) < 1e-10, ("state change over an RK cycle", l, rel_l2(a, b))

    s = _device(prm0, [hb])
    try:
        cycles(s, prm0, 2)
        s.setParams(prm1)
        pre = s.downloadState(0)
        assert s.infChangeCorrection(list(prm0.wInf)[:5], 1e-12, kind)
        corrected = s.downloadState(0)
        cycles(s, prm1, 3)
        live = s.downloadState(0)
    finally:
        s.close()
    ref = hb.copy()
    ref.w[...], ref.p[...], ref.rlv[...], ref.rev[...] = pre
    IC.inf_change_correction([ref], prm1, list(prm0.wInf)[:5], kind=kind)
    assert_state(corrected, ref)
    fresh_hb = hb.copy()
    fresh_hb.w[...], fresh_hb.p[...], fresh_hb.rlv[...], fresh_hb.rev[...] = corrected
    f = _device(prm1, [fresh_hb])
    try:
        for _ in range(3):
            _cycle(f)
        fresh = f.downloadState(0)
    finally:
        f.close()
    for a, b in zip(live, fresh):
        assert np.array_equal(a, b)


def test_residual_after_correction_matches_oracle(cuda_lib):
    """nothing cached before the correction survives it: the full residual of the corrected state"""
    prm0, prm1 = IC.free_stream_pair("RANS", "alpha", 2)
    hb = case(*SHAPE)[1]
    s = _device(prm0, [hb])
    try:
        s.residual(RES_FLOW | RES_TURB)
        s.residual(RES_FLOW | RES_TURB)   # replayed graph
        s.setParams(prm1)
        assert s.infChangeCorrection(list(prm0.wInf)[:5], 1e-12, "rotate")
        state = s.downloadState(0)
        s.residual(RES_FLOW | RES_TURB)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ho = hb.copy()
    ho.w[...], ho.p[...], ho.rlv[...], ho.rev[...] = state
    import ctypes as C

    o = Oracle(ho, prm1)
    o.pressure(False); o.lam_viscosity(False); o.eddy_viscosity(False)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    d = ho.d
    o.L.orc_etot(C.byref(o.ob), C.byref(prm1), 2, d.il, 2, d.jl, 2, d.kl)
    o.residual_core(RES_FLOW | RES_TURB)
    ow = d.owned()
    for l in range(6):
        assert rel_l2(dw[ow + (l,)], ho.dw[ow + (l,)]) < 1e-12, l
