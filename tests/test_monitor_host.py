"""The numpy restatement of the monitor routines (tests/monitor_ref.py) against the reference's own sumResiduals,
sumAllResiduals, maxHdiffMach and maxEddyv, bit for bit; the stopping rules of solveState (solver.convergence_status)
on made-up histories; the monitorVariables names (solver.monitor_names)."""
import math

import numpy as np
import pytest

import monitor_ref as MR
from adflow_b200 import synthetic as syn
from adflow_b200.solver import convergence_status, monitor_names
from oracle.pyoracle import Oracle
from util import case, overset_layout

needs_ref = pytest.mark.skipif(not MR.available(), reason="the reference source or oracle/_ref is not present")


def _blocks(eq, level):
    """three blocks of different shapes on `level`; level 2: the coarse blocks of level-1 blocks, with a made-up dw"""
    out = []
    for q, sh in enumerate(((10, 8, 6), (7, 9, 8), (12, 6, 7))):
        prm, hb = case(*sh, {"equationType": eq}, seed=200 + q)
        if q == 1:
            overset_layout(hb, at=(3, 3, 3))
        if level == 1:
            Oracle(hb, prm).residual_core(8 | 16)
        else:
            hb = syn.make_coarse_block(hb, prm)
            hb.dw[...] = np.random.default_rng(q).standard_normal(hb.dw.shape)
        out.append(hb)
    return prm, out


@needs_ref
@pytest.mark.parametrize("level", [1, 2])
@pytest.mark.parametrize("eq", ["Euler", "laminar NS", "RANS"])
def test_restatement_is_the_reference(eq, level):
    prm, blocks = _blocks(eq, level)
    # the largest Mach number, enthalpy difference and eddy-viscosity ratio in a halo-adjacent owned cell of the last block
    last = blocks[-1]
    il = last.d.il
    last.w[il, 2, 3, 1] = 3.0 * max(np.abs(hb.w[..., 1]).max() for hb in blocks)
    last.w[il, 2, 3, 4] = 3.0 * max(np.abs(hb.w[..., 4]).max() for hb in blocks)
    last.rev[il, 2, 3] = 50.0 * np.abs(last.rev).max() + 1.0
    want = MR.reference_monitor(blocks, prm)
    got = MR.monitor_sums(blocks, prm)
    assert np.array_equal(got, want), (got, want)
    assert got[6] > 0 and got[7] > 0 and got[8] > 0 and (got[5] > 0) == (eq == "RANS") and (got[9] > 0) == (eq == "RANS")
    # the maxima come from that cell of the last block
    assert np.array_equal(MR.monitor_sums(blocks[-1:], prm, 2)[7:], got[7:])
    w = last.w[last.d.owned()]
    mach2 = (w[..., 1] ** 2 + w[..., 2] ** 2 + w[..., 3] ** 2) * w[..., 0] / (prm.gammaInf * last.p[last.d.owned()])
    assert np.unravel_index(np.argmax(mach2), mach2.shape) == (il - 2, 0, 1)
    for what in (1, 2):
        part = MR.monitor_sums(blocks, prm, what)
        assert np.array_equal(part[:7] if what == 1 else part[7:], got[:7] if what == 1 else got[7:])
        assert not (part[7:] if what == 1 else part[:7]).any()


def test_nan_makes_the_sums_nan():
    prm, hb = case(8, 7, 6)
    Oracle(hb, prm).residual_core(8 | 16)
    hb.dw[4, 3, 3, 2] = np.nan
    m = MR.monitor_sums([hb], prm, 1)
    assert math.isnan(m[2]) and math.isnan(m[6]) and not math.isnan(m[0])


# ---------------------------------------------------------------------------------------------------------------------
# stopping rules
def _status(ground, its, total_r, rho_res=1.0, n_cycles=10, values=None, **opts):
    vals = [rho_res, total_r] if values is None else values
    return convergence_status(ground, its, n_cycles, vals, rho_res, 2.0, total_r, 1.0, 4.0, **opts)


def test_coarse_rule_against_rho_res_start():
    # rhoRes < L2ConvergenceCoarse * rhoResStart (= 2)
    assert _status(2, 3, total_r=1e-30, rho_res=0.019, L2ConvergenceCoarse=1e-2) == (True, False)
    assert _status(2, 3, total_r=1e-30, rho_res=0.021, L2ConvergenceCoarse=1e-2) == (False, False)
    # totalR plays no part above level 1, nor do the cycles running out
    assert _status(3, 10, total_r=1e30, rho_res=0.021, L2ConvergenceCoarse=1e-2, maxL2DeviationFactor=1.0) == (False, False)


def test_absolute_and_relative_fine_rules():
    # totalR0 = 1, totalRStart = 4
    assert _status(1, 3, total_r=0.9e-3, L2Convergence=1e-3) == (True, False)
    assert _status(1, 3, total_r=1.1e-3, L2Convergence=1e-3) == (False, False)
    assert _status(1, 3, total_r=0.039, L2Convergence=1e-8, L2ConvergenceRel=1e-2) == (True, False)
    assert _status(1, 3, total_r=0.041, L2Convergence=1e-8, L2ConvergenceRel=1e-2) == (False, False)
    # rhoRes plays no part on level 1
    assert _status(1, 3, total_r=1.0, rho_res=1e-30, L2Convergence=1e-8, L2ConvergenceCoarse=1.0) == (False, False)


def test_default_relative_tolerance_never_triggers():
    assert _status(1, 3, total_r=4.0 * 1e-15, L2Convergence=1e-20, L2ConvergenceRel=1e-16) == (False, False)
    assert _status(1, 3, total_r=1e-300, L2Convergence=0.0, L2ConvergenceRel=1e-16) == (True, False)


def test_deviation_failure_only_on_level_one_when_the_cycles_ran_out():
    opts = dict(L2Convergence=1e-8, maxL2DeviationFactor=10.0)
    # totalR = 2e-7 > 10 * 1 * 1e-8
    assert _status(1, 9, total_r=2e-7, **opts) == (False, False)       # cycles left
    assert _status(1, 10, total_r=2e-7, **opts) == (False, True)       # nCycles spent
    assert _status(1, 12, total_r=2e-7, **opts) == (False, True)
    assert _status(1, 10, total_r=0.9e-7, **opts) == (False, False)    # within the factor
    assert _status(2, 10, total_r=2e-7, rho_res=1.0, **opts) == (False, False)
    # a relative convergence on the last cycle can come with the deviation failure, as in the reference
    assert _status(1, 10, total_r=2e-7, L2Convergence=1e-8, L2ConvergenceRel=1e-6, maxL2DeviationFactor=10.0) == (True, True)


@pytest.mark.parametrize("ground", [1, 2])
@pytest.mark.parametrize("at", [0, 1, 2])
def test_nan_in_any_monitored_value_fails(ground, at):
    vals = [0.5, 0.25, 0.125]
    vals[at] = float("nan")
    conv, failed = _status(ground, 1, total_r=0.25, values=vals, L2Convergence=1e-3)
    assert failed and not conv


# ---------------------------------------------------------------------------------------------------------------------
# monitorVariables
def test_monitor_names():
    assert monitor_names(["cpu", "resrho", "resturb"], True) == (["RSDMassRMS", "RSDTurbulentSANuTildeRMS", "totalR"], True)
    assert monitor_names(["resturb", "eddyv"], False) == (["RSDMassRMS", "totalR"], False)
    names, cpu = monitor_names(["MACH", "hdiff", "resmom", "resrhoe", "totalr", "eddyv"], True)
    assert names == ["RSDMassRMS", "RSDMomentumXRMS", "RSDMomentumYRMS", "RSDMomentumZRMS", "RSDEnergyStagnationDensityRMS",
                     "totalR", "MaxDiffHAndHinf", "MaxMach", "MaxRatioEddyAndLaminarViscosity"] and not cpu


@pytest.mark.parametrize("name", ["cl", "cd", "clp", "clv", "cdp", "cdv", "cfx", "cfy", "cfz", "cmx", "cmy", "cmz"])
def test_force_monitors_are_refused_with_the_alternative(name):
    with pytest.raises(ValueError, match="evalFunctions"):
        monitor_names(["resrho", name], True)


@pytest.mark.parametrize("name", ["yplus", "sepsensor", "cavitation", "axismoment", "nonsense"])
def test_other_monitors_are_refused(name):
    with pytest.raises(ValueError, match=name):
        monitor_names([name], True)
