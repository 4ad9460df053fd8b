"""Multigrid on the device (adfb_mg_restrict / adfb_mg_prolong / adfb_mg_cycle and the coarse-level branches of the
smoother entry points) against the oracle, which is pinned bit for bit against the reference's multiGrid.F90
(tests/test_oracle_vs_reference_mg.py).  Tolerances as in test_smoother_parity.py: 1e-12 on residual-like arrays,
1e-10 on state changes over a smoother cycle."""
import numpy as np
import pytest

from adflow_b200 import synthetic as syn
from adflow_b200.solver import ADFLOW_B200
from oracle.pyoracle import Oracle

from util import case, rel_l2, rel_max

pytestmark = pytest.mark.gpu


def make_levels(shape, options, nlev):
    prm, fine = case(*shape, options)
    o = Oracle(fine, prm)
    o.apply_turb_bc(True); o.apply_flow_bc(True)
    levels = [fine]
    for _ in range(nlev - 1):
        levels.append(syn.make_coarse_block(levels[-1], prm))
    return prm, levels


def oracle_transfer_to_coarse(prm, fine, coarse):
    of, oc = Oracle(fine, prm), Oracle(coarse, prm)
    of.time_step(False)
    of.residual_block(prm.cdisRK[0])
    oc.mg_restrict(of)
    oc.apply_flow_bc(False)
    oc.time_step(True)
    oc.mg_store_w1()
    oc.residual_block_coarse(prm.cdisRK[0], init=0)
    oc.mg_forcing()


def oracle_mg_cycle(prm, levels, cycling, dadi_subiter=0):
    """executeMGCycle (multiGrid.F90:825-955), ground level 1, one block per level; dadi_subiter > 0: DADISmoother
    with that many sub-iterations instead of RungeKuttaSmoother"""
    lv = 0
    for n, c in enumerate(cycling):
        if c == -1:
            lv -= 1
            of, oc = Oracle(levels[lv], prm), Oracle(levels[lv + 1], prm)
            of.mg_prolong(oc)
            of.apply_flow_bc(lv == 0)
        elif c == 0:
            o = Oracle(levels[lv], prm)
            if n > 0 and cycling[n - 1] != 1:
                o.time_step(True)
                o.residual_block(prm.cdisRK[0])
            if dadi_subiter:
                for _ in range(dadi_subiter - 1):
                    o.dadi_step()
                    o.residual_block(1.0)
                o.dadi_step()
            else:
                o.rk_smoother()
        else:
            oracle_transfer_to_coarse(prm, levels[lv], levels[lv + 1])
            lv += 1
    o = Oracle(levels[0], prm)
    if prm.equations == 3:
        for _ in range(prm.nSubiterTurb):
            o.sa_block()
    o.time_step(True)
    o.residual_block(prm.cdisRK[0])


def device(prm, levels):
    s = ADFLOW_B200(prm)
    s.addBlock(levels[0])
    for q in range(1, len(levels)):
        s.addCoarseBlock(levels[q], q - 1)
    return s


def prepare_fine(o):
    o.time_step(True)
    o.hb.fw[...] = 0
    o.residual_block(o.prm.cdisRK[0])


@pytest.mark.parametrize("shape,options", [((16, 12, 10), None), ((13, 9, 7), None), ((12, 8, 8), {"equationType": "Euler"}),
                                           ((10, 12, 6), {"equationType": "laminar NS"}),
                                           ((12, 10, 8), {"coarseDiscretization": "central plus matrix dissipation"}),
                                           ((12, 10, 8), {"coarseDiscretization": "upwind"}),
                                           ((12, 10, 8), {"equationType": "Euler", "coarseDiscretization": "central plus matrix dissipation"}),
                                           ((12, 10, 8), {"equationType": "Euler", "coarseDiscretization": "upwind"})])
def test_restrict_smooth_prolong_match_oracle(cuda_lib, shape, options):
    prm, levels = make_levels(shape, options, 2)
    dev_levels = [l.copy() for l in levels]
    fine, coarse = levels
    s = device(prm, dev_levels)
    try:
        # --- transferToCoarseGrid
        oracle_transfer_to_coarse(prm, fine, coarse)
        s.mgRestrict(1)
        d = coarse.d
        ow = d.owned()
        c1 = (slice(1, d.ie + 1), slice(1, d.je + 1), slice(1, d.ke + 1))
        w, p, rlv, rev = s.downloadState(1)
        assert rel_max(w[c1][..., :5], coarse.w[c1][..., :5]) < 1e-13
        assert rel_max(p[c1], coarse.p[c1]) < 1e-13
        if prm.equations != 1:
            assert rel_max(rlv[c1], coarse.rlv[c1]) < 1e-13
        if prm.equations == 3:
            assert rel_max(rev[c1], coarse.rev[c1]) < 1e-13
        wr = s.downloadArray(1, "wr", 5)
        dw = s.downloadResidual(1)
        w1 = s.downloadArray(1, "w1", 5)
        for l in range(5):
            assert rel_l2(wr[ow + (l,)], coarse.wr[ow + (l,)]) < 1e-11, ("wr", l, rel_l2(wr[ow + (l,)], coarse.wr[ow + (l,)]))
            assert rel_l2(dw[ow + (l,)], coarse.dw[ow + (l,)]) < 1e-12, ("dw", l)
        assert rel_max(w1[c1], coarse.w1[c1]) < 1e-13
        assert rel_max(s.downloadArray(1, "dtl")[ow], coarse.dtl[ow]) < 1e-12
        # --- Runge-Kutta smoother on the coarse level
        w0 = coarse.w.copy()
        Oracle(coarse, prm).rk_smoother()
        s.rkCycle(level=2)
        w, p, rlv, rev = s.downloadState(1)
        for l in range(5):
            a, b = w[ow + (l,)] - w0[ow + (l,)], coarse.w[ow + (l,)] - w0[ow + (l,)]
            assert np.abs(b).max() > 0
            assert rel_l2(a, b) < 1e-9, ("coarse state change", l, rel_l2(a, b))
        assert rel_max(w[c1][..., :5], coarse.w[c1][..., :5]) < 1e-11
        # --- transferToFineGrid
        f0 = fine.w.copy()
        of, oc = Oracle(fine, prm), Oracle(coarse, prm)
        of.mg_prolong(oc)
        of.apply_flow_bc(True)
        s.mgProlong(1)
        w, p, rlv, rev = s.downloadState(0)
        owf = fine.d.owned()
        for l in range(5):
            a, b = w[owf + (l,)] - f0[owf + (l,)], fine.w[owf + (l,)] - f0[owf + (l,)]
            assert np.abs(b).max() > 0
            assert rel_l2(a, b) < 1e-9, ("fine correction", l, rel_l2(a, b))
        assert rel_max(w[..., :5], fine.w[..., :5]) < 1e-11
        assert rel_max(p, fine.p) < 1e-11
    finally:
        s.close()


@pytest.mark.parametrize("shape,options,cycle", [((16, 12, 8), None, "2v"), ((16, 16, 8), None, "3w"),
                                                 ((12, 12, 8), {"equationType": "Euler", "nRKStages": 3, "resAveraging": "never"}, "3v")])
def test_mg_cycle_matches_oracle(cuda_lib, shape, options, cycle):
    nlev = int(cycle[0])
    prm, levels = make_levels(shape, options, nlev)
    dev_levels = [l.copy() for l in levels]
    cyc = ADFLOW_B200.cycleStrategy(cycle)
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
        # a second cycle replays the captured graph
        s.mgCycle(cyc)
        w2, *_ = s.downloadState(0)
    finally:
        s.close()
    fine = levels[0]
    ow = fine.d.owned()
    for l in range(5):
        a, b = w[ow + (l,)] - w0[ow + (l,)], fine.w[ow + (l,)] - w0[ow + (l,)]
        assert np.abs(b).max() > 0
        assert rel_l2(a, b) < 1e-8, ("state change over the cycle", l, rel_l2(a, b))
        assert rel_l2(dw[ow + (l,)], fine.dw[ow + (l,)]) < 1e-8, ("residual after the cycle", l)
    assert rel_max(w[..., :5], fine.w[..., :5]) < 1e-10
    assert np.isfinite(w2).all() and np.abs(w2 - w).max() > 0


def test_mg_cycle_with_dadi_smoother(cuda_lib):
    prm, levels = make_levels((16, 12, 8), {"smoother": "DADI", "resAveraging": "never"}, 3)
    dev_levels = [l.copy() for l in levels]
    cyc = ADFLOW_B200.cycleStrategy("3w")
    prepare_fine(Oracle(levels[0], prm))
    w0 = levels[0].w.copy()
    oracle_mg_cycle(prm, levels, cyc, dadi_subiter=2)
    s = device(prm, dev_levels)
    try:
        s.timeStep(False)
        s.smootherResidual(0)
        s.mgCycle(cyc, smoother="DADI", n_subiterations=2)
        w, p, rlv, rev = s.downloadState(0)
    finally:
        s.close()
    fine = levels[0]
    ow = fine.d.owned()
    for l in range(5):
        a, b = w[ow + (l,)] - w0[ow + (l,)], fine.w[ow + (l,)] - w0[ow + (l,)]
        assert np.abs(b).max() > 0
        assert rel_l2(a, b) < 1e-7, ("state change over the cycle", l, rel_l2(a, b))
    assert rel_max(w[..., :5], fine.w[..., :5]) < 1e-9


@pytest.mark.parametrize("shape,options", [((16, 12, 8), None), ((12, 8, 8), {"equationType": "Euler"})])
def test_full_multigrid_start_up(cuda_lib, shape, options):
    """solver loop of src/solver/solvers.F90:63-117 with mgStartlevel = 2: single-grid cycles on ground level 2 (fine-grid
    routines on the coarse block, cflCoarse, second halos, turbulence solve), then transferToFineGrid(.false.).  The oracle
    composition is pinned bit for bit against the reference in tests/test_oracle_vs_reference_mg.py
    (test_rk_smoother_on_a_coarse_ground_level, test_full_multigrid_start_up_transfer)."""
    prm, levels = make_levels(shape, options, 2)
    fine, coarse = levels
    # a coarse start solution with halos; the fine state is whatever the start-up finds there (it is overwritten)
    oracle_transfer_to_coarse(prm, fine, coarse)
    dev_levels = [l.copy() for l in levels]
    n_cycles = 2
    cfl = prm.cfl
    try:                                     # oracle: the coarse block as a ground level = level-1 semantics with cflCoarse
        prm.cfl = prm.cflCoarse
        coarse.level = 1
        og = Oracle(coarse, prm)
        if prm.equations == 3:
            og.apply_turb_bc(True)
        og.apply_flow_bc(True)
        og.time_step(True)
        coarse.fw[...] = 0
        og.residual_block(prm.cdisRK[0])
        c0 = coarse.w.copy()
        for _ in range(n_cycles):
            oracle_mg_cycle(prm, [coarse], [0])
    finally:
        prm.cfl = cfl
        coarse.level = 2
    cs = coarse.copy()                       # the transfer overwrites the coarse rho*E and boundary halos
    of, oc = Oracle(fine, prm), Oracle(coarse, prm)
    of.mg_prolong_solution(oc)
    if prm.equations == 3:
        of.apply_turb_bc(True)
    of.apply_flow_bc(True); of.apply_flow_bc(True); of.apply_flow_bc(True)
    s = device(prm, dev_levels)
    try:
        s.setGroundLevel(2)
        s.applyBCs(True, True, level=2)
        s.timeStep(False, level=2)
        s.smootherResidual(0, level=2)
        for _ in range(n_cycles):
            s.mgCycle([0])
        wc, pc, _, revc = s.downloadState(1)
        from adflow_b200._lib import AdflowB200Error
        with pytest.raises(AdflowB200Error):
            s.mgProlongSolution(2)           # no level 3 / wrong ground level
        s.mgProlongSolution(1)
        s.setGroundLevel(1)
        w, p, rlv, rev = s.downloadState(0)
        # the fine level is usable right away: one residual on it
        s.timeStep(False); s.smootherResidual(0)
        dw = s.downloadResidual(0)
    finally:
        s.close()
    ow = coarse.d.owned()
    # coarse ground level after the cycles
    assert rel_max(wc[..., :5], cs.w[..., :5]) < 1e-9
    assert rel_max(pc, cs.p) < 1e-9
    assert np.abs(cs.w[ow][..., :5] - c0[ow][..., :5]).max() > 0
    assert rel_max(w, fine.w) < 1e-9, rel_max(w, fine.w)
    assert rel_max(p, fine.p) < 1e-9
    if prm.equations != 1:
        assert rel_max(rlv, fine.rlv) < 1e-9
    if prm.equations == 3:
        assert rel_max(rev, fine.rev) < 1e-8
    o = Oracle(fine, prm)
    o.time_step(True); fine.fw[...] = 0; o.residual_block(prm.cdisRK[0])
    owf = fine.d.owned()
    for l in range(5):
        assert rel_l2(dw[owf + (l,)], fine.dw[owf + (l,)]) < 1e-7, ("fine residual after the start-up", l)


def test_cycle_strategy_and_errors(cuda_lib):
    assert ADFLOW_B200.cycleStrategy("sg") == [0]
    assert ADFLOW_B200.cycleStrategy("2v") == [0, 1, 0, -1]
    assert len(ADFLOW_B200.cycleStrategy("4w")) == 28      # computeNstepsWcycle(4) = 4 + 2 * (4 + 2 * 4)
    prm, levels = make_levels((8, 8, 6), None, 2)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(levels[0])
        from adflow_b200._lib import AdflowB200Error
        with pytest.raises(AdflowB200Error):
            s.mgRestrict(1)                 # no coarse level
        s.addBlock(levels[1], level=2)      # coarse block without tables
        with pytest.raises(AdflowB200Error):
            s.mgRestrict(1)
        with pytest.raises(AdflowB200Error):
            s.mgCycle([0, 1, 0])            # does not return to the ground level
    finally:
        s.close()


def test_two_block_v_cycle_with_halo_exchange_per_level(cuda_lib):
    """2 blocks per level on one GPU: transferToCoarseGrid / the coarse RK stages / transferToFineGrid with the
    exchange of each level's own pattern (whalo1 on level 2) between the per-block operations."""
    from adflow_b200 import make_params
    from adflow_b200.halo import BlockGrid, build_cartesian_pattern, comm_vars, exchange_numpy, make_grid_blocks

    prm = make_params({"equationType": "laminar NS", "nRKStages": 3, "resAveraging": "never"})
    gf = BlockGrid((2, 1, 1), (8, 8, 6), nranks=1)
    fine = make_grid_blocks(gf, 0, prm)
    pf = build_cartesian_pattern(gf, 0)
    vars_ = lambda hb: comm_vars(hb, 1, 5, True, True, True, False)  # noqa: E731
    for hb in fine:
        o = Oracle(hb, prm)
        o.apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)
    coarse = [syn.make_coarse_block(hb, prm) for hb in fine]
    gc = BlockGrid((2, 1, 1), (4, 4, 3), nranks=1)
    pc = build_cartesian_pattern(gc, 0)
    dev_f, dev_c = [b.copy() for b in fine], [b.copy() for b in coarse]

    def rk_smoother(blocks, pat, second):
        for hb in blocks:
            np.copyto(hb.wn, hb.w[..., :5]); np.copyto(hb.pn, hb.p)
        for st in range(1, prm.nRKStages + 1):
            for hb in blocks:
                Oracle(hb, prm).rk_stage(st)
            exchange_numpy(blocks, pat, vars_)
            if st < prm.nRKStages:
                for hb in blocks:
                    Oracle(hb, prm).residual_block(prm.cdisRK[st])

    # the fine residual the cycle starts from
    for hb in fine:
        prepare_fine(Oracle(hb, prm))
    w0 = [hb.w.copy() for hb in fine]
    # executeMGCycle for 2v = 0 1 0 -1 (+ timeStep, residual at the end)
    rk_smoother(fine, pf, True)
    for f, c in zip(fine, coarse):
        of, oc = Oracle(f, prm), Oracle(c, prm)
        of.time_step(False); of.residual_block(prm.cdisRK[0])
        oc.mg_restrict(of); oc.apply_flow_bc(False)
    exchange_numpy(coarse, pc, vars_)
    for c in coarse:
        oc = Oracle(c, prm)
        oc.time_step(True); oc.mg_store_w1(); oc.residual_block_coarse(prm.cdisRK[0], init=0); oc.mg_forcing()
    rk_smoother(coarse, pc, False)
    for f, c in zip(fine, coarse):
        of, oc = Oracle(f, prm), Oracle(c, prm)
        of.mg_prolong(oc); of.apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)
    for f in fine:
        o = Oracle(f, prm)
        o.time_step(True); o.residual_block(prm.cdisRK[0])

    s = ADFLOW_B200(prm)
    try:
        for hb in dev_f:
            s.addBlock(hb)
        for q, hb in enumerate(dev_c):
            s.addCoarseBlock(hb, q)
        s.setCommPattern(pf, level=1)
        s.setCommPattern(pc, level=2, block_offset=2)
        s.timeStep(False)
        s.smootherResidual(0)
        s.mgCycle(ADFLOW_B200.cycleStrategy("2v"))
        for q, hb in enumerate(fine):
            w, p, rlv, rev = s.downloadState(q)
            dw = s.downloadResidual(q)
            ow = hb.d.owned()
            for l in range(5):
                a, b = w[ow + (l,)] - w0[q][ow + (l,)], hb.w[ow + (l,)] - w0[q][ow + (l,)]
                assert np.abs(b).max() > 0
                assert rel_l2(a, b) < 1e-8, (q, l, rel_l2(a, b))
                assert rel_l2(dw[ow + (l,)], hb.dw[ow + (l,)]) < 1e-8, (q, l)
            assert rel_max(w[..., :5], hb.w[..., :5]) < 1e-10, q    # halos incl. the exchanged ones
    finally:
        s.close()


def _mg_nccl_worker(rank, world, port, q):
    import ctypes as C
    import os

    import torch
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from adflow_b200 import _lib, make_params
    from adflow_b200.halo import BlockGrid, build_cartesian_pattern, make_grid_blocks
    L = _lib.load()
    uid = torch.zeros(128, dtype=torch.uint8)
    if rank == 0:
        buf = (C.c_char * 128)()
        assert L.adfb_get_unique_id(buf) == 0
        uid = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8).clone()
    dist.broadcast(uid, 0)
    prm = make_params(_TWO_GPU_OPTS)
    gf = BlockGrid((2, 1, 1), _TWO_GPU_SHAPE, nranks=world)
    fine = make_grid_blocks(gf, rank, prm)
    gc = BlockGrid((2, 1, 1), tuple(n // 2 for n in _TWO_GPU_SHAPE), nranks=world)
    s = ADFLOW_B200(prm, device=rank, rank=rank, nranks=world, unique_id=bytes(uid.numpy().tobytes()))
    for hb in fine:
        s.addBlock(hb)
    for qb, hb in enumerate(fine):
        s.addCoarseBlock(syn.make_coarse_block(hb, prm), qb)
    s.setCommPattern(build_cartesian_pattern(gf, rank), level=1)
    s.setCommPattern(build_cartesian_pattern(gc, rank), level=2, block_offset=len(fine))
    s.applyBCs(True, False)
    s.haloExchange(1, 5, True, True, True)
    s.timeStep(False)
    s.smootherResidual(0)
    s.mgCycle(ADFLOW_B200.cycleStrategy("2v"))
    out = {}
    for lq, b in enumerate(gf.local_blocks(rank)):
        out[b] = s.downloadState(lq)[0]
    s.close()
    q.put((rank, out))
    dist.barrier()
    dist.destroy_process_group()


_TWO_GPU_OPTS = {"equationType": "laminar NS", "nRKStages": 3, "resAveraging": "never"}
_TWO_GPU_SHAPE = (8, 8, 6)


def test_two_gpu_v_cycle_matches_single_process_oracle(cuda_lib):
    """one fine + one coarse block per GPU, NCCL exchange of each level's pattern inside the multigrid cycle"""
    if cuda_lib.adfb_device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import os

    import torch.multiprocessing as mp
    from adflow_b200 import make_params
    from adflow_b200.halo import BlockGrid, build_cartesian_pattern, comm_vars, exchange_numpy, make_grid_blocks

    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29900 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_mg_nccl_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    got = {}
    for _ in range(world):
        _rank, out = q.get(timeout=600)
        got.update(out)
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    # the same cycle with the oracle, all blocks in one process
    prm = make_params(_TWO_GPU_OPTS)
    gf = BlockGrid((2, 1, 1), _TWO_GPU_SHAPE, nranks=1)
    fine = make_grid_blocks(gf, 0, prm)
    pf = build_cartesian_pattern(gf, 0)
    coarse = [syn.make_coarse_block(hb, prm) for hb in fine]
    pc = build_cartesian_pattern(BlockGrid((2, 1, 1), tuple(n // 2 for n in _TWO_GPU_SHAPE), nranks=1), 0)
    vars_ = lambda hb: comm_vars(hb, 1, 5, True, True, True, False)  # noqa: E731

    def rk_smoother(blocks, pat):
        for hb in blocks:
            np.copyto(hb.wn, hb.w[..., :5]); np.copyto(hb.pn, hb.p)
        for st in range(1, prm.nRKStages + 1):
            for hb in blocks:
                Oracle(hb, prm).rk_stage(st)
            exchange_numpy(blocks, pat, vars_)
            if st < prm.nRKStages:
                for hb in blocks:
                    Oracle(hb, prm).residual_block(prm.cdisRK[st])

    for hb in fine:
        Oracle(hb, prm).apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)
    w0 = [hb.w.copy() for hb in fine]
    for hb in fine:
        prepare_fine(Oracle(hb, prm))
    rk_smoother(fine, pf)
    for f, c in zip(fine, coarse):
        of, oc = Oracle(f, prm), Oracle(c, prm)
        of.time_step(False); of.residual_block(prm.cdisRK[0])
        oc.mg_restrict(of); oc.apply_flow_bc(False)
    exchange_numpy(coarse, pc, vars_)
    for c in coarse:
        oc = Oracle(c, prm)
        oc.time_step(True); oc.mg_store_w1(); oc.residual_block_coarse(prm.cdisRK[0], init=0); oc.mg_forcing()
    rk_smoother(coarse, pc)
    for f, c in zip(fine, coarse):
        of, oc = Oracle(f, prm), Oracle(c, prm)
        of.mg_prolong(oc); of.apply_flow_bc(True)
    exchange_numpy(fine, pf, vars_)
    for b, hb in enumerate(fine):
        ow = hb.d.owned()
        for l in range(5):
            a, r = got[b][ow + (l,)] - w0[b][ow + (l,)], hb.w[ow + (l,)] - w0[b][ow + (l,)]
            assert np.abs(r).max() > 0
            assert rel_l2(a, r) < 1e-8, (b, l, rel_l2(a, r))
        assert rel_max(got[b][..., :5], hb.w[..., :5]) < 1e-10, b


def test_multigrid_accelerates_convergence_like_the_oracle(cuda_lib):
    """ten cycles, Euler: the density-residual history of the device follows the oracle's cycle by cycle, and the
    3W cycle converges about twice as fast per cycle as the single-grid smoother (what multigrid is for)"""
    opts = {"equationType": "Euler"}
    hist = {}
    for name, nlev in (("sg", 1), ("3w", 3)):
        prm, levels = make_levels((16, 16, 8), opts, nlev)
        dev_levels = [l.copy() for l in levels]
        cyc = ADFLOW_B200.cycleStrategy(name)
        prepare_fine(Oracle(levels[0], prm))
        ref = [Oracle(levels[0], prm).norms()[0]]
        for _ in range(10):
            oracle_mg_cycle(prm, levels, cyc)
            ref.append(Oracle(levels[0], prm).norms()[0])
        s = device(prm, dev_levels)
        try:
            s.timeStep(False)
            s.smootherResidual(0)
            got = [s.getResNorms()[0]]
            for _ in range(10):
                s.mgCycle(cyc)
                got.append(s.getResNorms()[0])
        finally:
            s.close()
        ref, got = np.sqrt(ref), np.sqrt(got)
        assert np.allclose(got, ref, rtol=1e-7, atol=0), (name, np.abs(got / ref - 1).max())
        hist[name] = got
    assert hist["3w"][-1] < 0.6 * hist["sg"][-1], (hist["3w"][-1], hist["sg"][-1])
    assert hist["sg"][-1] < hist["sg"][0]
