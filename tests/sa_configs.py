"""Thread tiles and k chunks of the SA-row tile kernel k_sa (adflow_b200/csrc/sa_tile.cuh) that both the CPU emulation
(tests/test_sa_emul.py) and the device (tests/test_sa_tile_gpu.py) run, so that a failure on the device alone points at
code only the device runs (cp.async groups, barriers, the plane ring), and the comparisons both use.

The blocks have partial tiles in i and j.  The k chunks cover one plane (no carry at all), short chunks with several
seams, the whole plane range in one chunk or one short of it, and the chunks sa_tile_choose picks for the bench-sized
blocks on an H100 (132 SMs, 3 resident CTAs each), where every CTA carries its column through many planes."""
import numpy as np

from util import rel_l2

SHAPES = [(37, 13, 17), (33, 9, 23)]
TILES = [(32, 4), (16, 8), (7, 4), (5, 7)]
# block -> (TX, TY, kChunk) of sa_tile_choose on 132 SMs with 3 CTAs each (C2 block, one C3 block, one C5 block); 3 is what the
# occupancy query gives k_sa on an H100 (the k_sa grid of a one-tile block under ADFB_SM_COUNT=1 has 3 k chunks)
BENCH_PICKS = {(96, 72, 64): (16, 8, 10), (128, 128, 64): (16, 8, 22), (160, 160, 144): (16, 8, 144)}
H100_SMS, SA_CTAS_PER_SM = 132, 3

# the SA options of the emulation and device tests
OPTIONS = [{"turbulenceOrder": "second order"}, {"turbulenceProduction": "vorticity"}, {"useRotationSA": True}, {"useft2SA": False},
           {"useApproxSA": True}, {"turbulenceOrder": "second order", "turbulenceProduction": "vorticity", "useft2SA": False}]


def chunks(n_planes):
    """the k chunks of the matrix for a block of n_planes owned planes (clamped to n_planes, as ADFB_SA_TILE is)"""
    want = [1, 2, 3, 5, n_planes - 1, n_planes] + [p[2] for p in BENCH_PICKS.values()]
    return sorted({min(max(c, 1), n_planes) for c in want})


CONFIGS = [(shape, (tx, ty, kc)) for shape in SHAPES for tx, ty in TILES for kc in chunks(shape[2])]


def config_id(c):
    shape, tile = c
    return "%s-%s" % ("x".join(map(str, shape)), "x".join(map(str, tile)))


def sa_tile_choose(shape, n_planes, n_sm, ctas_per_sm):
    """sa_tile_choose restated: 32 x 4 or 16 x 8, whichever loads fewer halo cells, then the longest k chunk that still
    fills every resident CTA slot once"""
    nx, ny = shape[0], shape[1]
    best = None
    for tx, ty in ((32, 4), (16, 8)):
        cost = -(-nx // tx) * -(-ny // ty) * (tx + 2) * (ty + 2)
        if best is None or cost < best[0]:
            best = (cost, tx, ty)
    _, tx, ty = best
    tiles = -(-nx // tx) * -(-ny // ty)
    n = min(max(n_sm * ctas_per_sm // tiles, 1), n_planes)
    return tx, ty, max(-(-n_planes // n), 1)


def sa_grid(shape, n_planes, tile):
    """grid and block of the k_sa launch for a tile (TX, TY, kChunk)"""
    tx, ty, kc = tile
    return (-(-shape[0] // tx), -(-shape[1] // ty), -(-n_planes // kc)), (tx * ty, 1, 1)


def assert_sa_planes(got, want, plane_tol=1e-11, l2_tol=1e-12, what="SA row"):
    """got / want: the SA row of the owned cells, k last.  Plane by plane, max|got - want| <= plane_tol x max|want| of that
    plane (an error confined to one plane cannot hide behind the rest of the row), and rel L2 of the row < l2_tol."""
    assert np.isfinite(got).all(), what
    for k in range(want.shape[-1]):
        e, m = np.abs(got[..., k] - want[..., k]).max(), np.abs(want[..., k]).max()
        assert e <= plane_tol * m, "%s, owned plane %d: max|d| %.3e, max|ref| %.3e" % (what, k, e, m)
    assert rel_l2(got, want) < l2_tol, "%s: rel L2 %.3e" % (what, rel_l2(got, want))
