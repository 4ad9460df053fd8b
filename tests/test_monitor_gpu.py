"""The convergence monitor (adfb_monitor) against its numpy restatement (tests/monitor_ref.py, pinned bit for bit to the
reference's own routines in tests/test_monitor_host.py), adfb_norms against the monitor, and solveState / solve against
the same loop composed from the oracle's cycles (test_mg_gpu.oracle_mg_cycle, tests/fmg_oracle.py).

Tolerances: the sums 1e-13 relative (the device reduces in another order), the maxima bit for bit; the monitored values
of a solver history 1e-7, as test_mg_gpu.py's convergence history.  Every test that compares a stopping iteration first
shows on the oracle's history that the stopping iteration lies at least 5 % below its threshold and every iteration
before it at least 5 % above, so that rounding cannot decide the stop."""
import ctypes as C
import math

import numpy as np
import pytest

import diss_continuation as DC
import fmg_oracle as F
import monitor_ref as MR
from adflow_b200._lib import AdflowB200Error
from adflow_b200.halo import BlockGrid, build_cartesian_pattern, make_grid_blocks
from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
from oracle.pyoracle import Oracle
from test_mg_gpu import device, make_levels, oracle_mg_cycle
from util import case, overset_layout

pytestmark = pytest.mark.gpu

FT = RES_FLOW | RES_TURB
EQS = ["Euler", "laminar NS", "RANS"]


def _host_blocks(s, ids):
    """the device's blocks `ids` as HostBlocks holding the device's w, p, rlv, rev and dw"""
    out = []
    for b in ids:
        hb = s.blocks[b].copy()
        hb.w[...], hb.p[...], hb.rlv[...], hb.rev[...] = s.downloadState(b)
        hb.dw[...] = s.downloadResidual(b)
        out.append(hb)
    return out


def _check(got, want, what):
    sums = [q for q in range(7) if what & 1]
    for q in sums:
        assert abs(got[q] - want[q]) <= 1e-13 * abs(want[q]), (q, got[q], want[q])
    for q in range(7, 10):
        if what & 2:
            assert got[q] == want[q], (q, got[q], want[q])
        else:
            assert got[q] == 0.0
    if not what & 1:
        assert not got[:7].any()


@pytest.mark.parametrize("what", [1, 2, 3])
@pytest.mark.parametrize("eq", EQS)
def test_monitor_of_each_level(cuda_lib, eq, what):
    """levels 1, 2, 3 of one context: each level's blocks only, after a residual on that ground level"""
    prm, levels = make_levels((16, 12, 10), {"equationType": eq}, 3)
    s = device(prm, [l.copy() for l in levels])
    try:
        for lv in (3, 2, 1):
            s.setGroundLevel(lv)
            s.residual(FT, level=lv)
            got = s.monitorSums(lv, what)
            want = MR.monitor_sums(_host_blocks(s, [lv - 1]), prm, what)
            full = MR.monitor_sums(_host_blocks(s, [lv - 1]), prm)
            assert full[6] > 0 and full[8] > 0 and (eq != "RANS" or lv > 1 or full[9] > 0)
            _check(got, want, what)
            assert np.array_equal(s.monitorSums(lv, what), got)     # the same bits on every call
    finally:
        s.close()


@pytest.mark.parametrize("what", [1, 2, 3])
@pytest.mark.parametrize("eq", EQS)
def test_monitor_of_several_blocks(cuda_lib, eq, what):
    """two blocks with a 1-to-1 pattern, four blocks of different shapes, one of them blanked (tests/util.py); the
    largest values sit in the last block"""
    opts = {"equationType": eq}
    prm, _ = case(8, 8, 6, opts)
    grid = BlockGrid((2, 1, 1), (8, 8, 6), nranks=1)
    blocks = make_grid_blocks(grid, 0, prm)
    for q, sh in enumerate(((12, 10, 8), (9, 14, 6), (7, 8, 11), (10, 9, 9))):
        hb = case(*sh, opts, seed=100 + q)[1]
        if q == 2:
            overset_layout(hb)
        blocks.append(hb)
    last = blocks[-1]
    # a halo-adjacent owned cell (i = 2) of the last block: the largest speed, at the same pressure
    u = 1.5 * max(np.abs(hb.w[..., 1]).max() for hb in blocks)
    last.w[2, 3, 4, 4] += 0.5 * last.w[2, 3, 4, 0] * (u * u - last.w[2, 3, 4, 1] ** 2)
    last.w[2, 3, 4, 1] = u
    s = ADFLOW_B200(prm)
    try:
        for hb in blocks:
            s.addBlock(hb)
        s.setCommPattern(build_cartesian_pattern(grid, 0), level=1)
        s.residual(FT)
        got = s.monitorSums(1, what)
        host = _host_blocks(s, range(len(blocks)))
        want = MR.monitor_sums(host, prm, what)
        if what & 2:
            assert want[8] == MR.monitor_sums(host[-1:], prm, 2)[8]
        _check(got, want, what)
    finally:
        s.close()


@pytest.mark.parametrize("eq", EQS)
def test_norms_are_the_monitor_sums(cuda_lib, eq):
    """adfb_norms is out[0] and out[6] of the level-1 monitor, bit for bit, and coarse blocks add nothing to it"""
    prm, levels = make_levels((16, 12, 10), {"equationType": eq}, 2)
    s = device(prm, [l.copy() for l in levels])
    try:
        s.residual(FT)
        m = s.monitorSums(1, 1)
        n = s.getResNorms()
        assert n[0] == m[0] and n[1] == m[6]
        want = MR.monitor_sums(_host_blocks(s, [0]), prm, 1)
        assert abs(n[1] - want[6]) <= 1e-13 * want[6]
    finally:
        s.close()


def test_monitor_refusals(cuda_lib):
    prm, hb = case(8, 8, 6)
    out = (C.c_double * 10)()
    s = ADFLOW_B200(prm)
    L = s.L

    def refused(*args):
        assert L.adfb_monitor(*args) != 0
        buf = C.create_string_buffer(1024)
        L.adfb_last_error(buf, 1024)
        assert b"adfb_monitor" in buf.value, buf.value

    try:
        refused(1, 3, out)                  # no block
        s.addBlock(hb)
        refused(1, 3, None)
        refused(1, 0, out)
        refused(1, 4, out)
        refused(1, 7, out)
        refused(2, 3, out)                  # no block of level 2
        with pytest.raises(ValueError):
            s.monitor(1, ["resrho", "cl"])
    finally:
        s.close()
    assert L.adfb_init(0, None, 0, 1) == 0
    try:
        refused(1, 3, out)                  # no parameters
    finally:
        L.adfb_finalize()


# ---------------------------------------------------------------------------------------------------------------------
# solveState and solve against the oracle's loop
def _values(prm, hb):
    m = MR.monitor_sums([hb], prm, 1)
    n = hb.d.nx * hb.d.ny * hb.d.nz
    return {"RSDMassRMS": math.sqrt(m[0] / n), "RSDTurbulentSANuTildeRMS": math.sqrt(m[5] / n), "totalR": math.sqrt(m[6])}


def oracle_ground(prm, levels, ground, cycle, n_cycles, dadi_subiter=0, totals=None):
    """solveState's iterations on ground level `ground` with the oracle, n_cycles of them without a stopping test; the
    monitored values per iteration.  totals: (totalR, totalR0) of the dissipation-based continuation, updated after
    each monitor (then prm is the parameters with continuation)."""
    hb = levels[ground - 1]

    def p():
        return prm if totals is None else DC.oracle_params(prm, *totals)

    g = F.Ground(hb, p())
    g.preamble()
    g.blockette_residual()
    if ground == 1:
        Oracle(hb, p()).time_step(True)
    else:
        g.time_step()
    hist = []
    cyc = ADFLOW_B200.cycleStrategy(cycle if ground == 1 else dict(ADFLOW_B200.fmgSchedule(ground, cycle))[ground])
    for it in range(n_cycles + 1):
        if it:
            if ground == 1:
                oracle_mg_cycle(p(), levels, cyc, dadi_subiter)
            else:
                F.mg_cycle(p(), levels[ground - 1:], cyc, dadi_subiter > 0)
        v = _values(prm, hb)
        hist.append(v)
        if totals is not None:
            totals[0] = v["totalR"]
    return hist


def pick_threshold(ratios, first=2):
    """a threshold t and the iteration s >= first at which ratios[s] < 0.95 t first, with ratios[i] > 1.05 t for every
    iteration 1 <= i < s"""
    for s in range(first, len(ratios)):
        before = min(ratios[1:s])
        if ratios[s] < before * (0.95 / 1.05):
            t = math.sqrt(before * ratios[s])
            assert ratios[s] < 0.95 * t and all(r > 1.05 * t for r in ratios[1:s])
            return t, s
    raise AssertionError("no iteration of the oracle history clears a threshold by 5 %%: %s" % (ratios,))


def _compare(hist, want, names, upto):
    assert hist["total minor iters"] == list(range(upto + 1))
    for name in names:
        got, ref = np.array(hist[name]), np.array([w[name] for w in want[:upto + 1]])
        assert np.allclose(got, ref, rtol=1e-7, atol=0), (name, np.abs(got / ref - 1).max())


def _free_stream_total(prm, hb):
    from test_oracle_vs_reference_diss_continuation import oracle_free_stream_residual

    return math.sqrt(oracle_free_stream_residual(prm, hb)[0][1])


@pytest.mark.parametrize("kind", ["Euler 3w RK", "RANS sg DADI"])
def test_solve_state_matches_the_oracle_loop(cuda_lib, kind):
    if kind.startswith("Euler"):
        prm, levels = make_levels((16, 16, 8), {"equationType": "Euler", "smoother": "Runge-Kutta"}, 3)
        cycle, smoother, nsub = "3w", "Runge-Kutta", 1
    else:
        prm, levels = make_levels((12, 10, 8), {"smoother": "DADI", "resAveraging": "never"}, 1)
        cycle, smoother, nsub = "sg", "DADI", 2
    dev_levels = [l.copy() for l in levels]
    tr0 = _free_stream_total(prm, levels[0])
    n = 14
    want = oracle_ground(prm, levels, 1, cycle, n, dadi_subiter=nsub if smoother == "DADI" else 0)
    if kind.startswith("Euler"):   # the absolute rule
        t, stop = pick_threshold([w["totalR"] / tr0 for w in want])
        opts = {"L2Convergence": t}
    else:                          # the relative rule
        t, stop = pick_threshold([w["totalR"] / want[0]["totalR"] for w in want])
        opts = {"L2Convergence": 1e-30, "L2ConvergenceRel": t}
    names = ["RSDMassRMS", "totalR"] + (["RSDTurbulentSANuTildeRMS"] if prm.equations == 3 else [])
    s = device(prm, dev_levels)
    try:
        r = s.solveState(nCycles=n, MGCycle=cycle, smoother=smoother, nSubiter=nsub, monitorVariables=["resrho", "resturb", "cpu"],
                         **opts)
        assert abs(s.totalR0 - tr0) <= 1e-10 * tr0
    finally:
        s.close()
    assert r["converged"] and not r["failed"]
    h = r["history"]
    assert len(h["totalR"]) == stop + 1, (len(h["totalR"]), stop)
    assert h["iter type"] == ["None"] + [("DADI" if smoother == "DADI" else "RK")] * stop
    assert len(h["wall time"]) == stop + 1
    _compare(h, want, names, stop)


def test_solve_from_level_three_matches_the_oracle_loop(cuda_lib):
    """solve(mg_start_level=3) with 3W: the coarse levels run out of their nCyclesCoarse cycles (L2ConvergenceCoarse far
    below their histories), level 1 stops on L2Convergence"""
    prm, levels = make_levels((16, 16, 8), {"equationType": "Euler", "smoother": "Runge-Kutta"}, 3)
    dev_levels = [l.copy() for l in levels]
    n_coarse, n = 3, 14
    coarse_tol = 1e-9
    want = {}
    for ground in (3, 2):
        want[ground] = oracle_ground(prm, levels, ground, "3w", n_coarse)
        F.prolong_solution(prm, levels[ground - 2], levels[ground - 1])
        assert all(w["RSDMassRMS"] > 1.05 * coarse_tol * want[ground][0]["RSDMassRMS"] for w in want[ground][1:])
    tr0 = _free_stream_total(prm, levels[0])
    want[1] = oracle_ground(prm, levels, 1, "3w", n)
    t, stop = pick_threshold([w["totalR"] / tr0 for w in want[1]])
    s = device(prm, dev_levels)
    try:
        s.setGroundLevel(3)
        out = s.solve(3, nCycles=n, nCyclesCoarse=n_coarse, L2Convergence=t, L2ConvergenceCoarse=coarse_tol, MGCycle="3w",
                      smoother="Runge-Kutta", monitorVariables=["resrho"])
        assert s.L.adfb_get_ground_level() == 1
    finally:
        s.close()
    assert [g for g, _ in out] == [3, 2, 1]
    for ground, r in out:
        h = r["history"]
        if ground > 1:
            assert not r["converged"] and not r["failed"]
            _compare(h, want[ground], ["RSDMassRMS", "totalR"], n_coarse)
            assert h["CFL"][1:] == [prm.cflCoarse] * n_coarse
        else:
            assert r["converged"] and not r["failed"] and len(h["totalR"]) == stop + 1
            _compare(h, want[1], ["RSDMassRMS", "totalR"], stop)


def test_solve_state_with_dissipation_based_continuation(cuda_lib):
    """useDissContinuation: every monitor passes totalR and totalR0 to the next residual, as iteration%totalR does"""
    import regimes as R

    prm, hb = R.regime_case("contact_pocket", (16, 12, 10), dict(DC.OPTIONS, equationType="Euler", resAveraging="never",
                                                                   smoother="Runge-Kutta"))
    Oracle(hb, prm).reference_shock_sensor()
    dev = hb.copy()
    tr0 = _free_stream_total(DC.oracle_params(prm, 0.0, 0.0), hb)
    n = 14
    totals = [0.0, tr0]
    want = oracle_ground(prm, [hb], 1, "sg", n, totals=totals)
    t, stop = pick_threshold([w["totalR"] / tr0 for w in want])
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(dev)
        r = s.solveState(nCycles=n, L2Convergence=t, smoother="Runge-Kutta", monitorVariables=["resrho"])
    finally:
        s.close()
    assert r["converged"] and len(r["history"]["totalR"]) == stop + 1
    _compare(r["history"], want, ["RSDMassRMS", "totalR"], stop)
    # without the continuation the history differs: the test reaches the coupling
    plain = oracle_ground(DC.plain(prm), [hb.copy()], 1, "sg", 2)
    assert plain[2]["totalR"] != want[2]["totalR"]


def test_solve_state_fails_on_nan_and_on_the_deviation_factor(cuda_lib):
    prm, levels = make_levels((12, 10, 8), {"equationType": "Euler", "smoother": "Runge-Kutta"}, 1)
    bad = levels[0].copy()
    bad.w[5, 4, 3, 0] = np.nan             # one owned cell's density
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(bad)
        r = s.solveState(nCycles=5, smoother="Runge-Kutta")
    finally:
        s.close()
    assert r["failed"] and not r["converged"]
    assert len(r["history"]["totalR"]) == 1 and math.isnan(r["history"]["totalR"][0])
    # the cycles run out on ground level 1 with totalR above maxL2DeviationFactor totalR0 L2Convergence
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(levels[0].copy())
        r = s.solveState(nCycles=2, L2Convergence=1e-12, maxL2DeviationFactor=10.0, smoother="Runge-Kutta")
        h = r["history"]
        assert r["failed"] and not r["converged"] and len(h["totalR"]) == 3
        assert h["totalR"][-1] > 10.0 * s.totalR0 * 1e-12 * 1.05
        with pytest.raises(AdflowB200Error):
            s.solveState(MGCycle="2v")       # no level 2 in this context
    finally:
        s.close()
