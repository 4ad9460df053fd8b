// sa_emul.cu -- CPU emulation of the SA-row tile kernel k_sa (adflow_b200/csrc/sa_tile.cuh).
// TEST INFRASTRUCTURE ONLY: runs the kernel's own per-thread phase functions (sa_prologue, sa_own_loads, sa_load_plane,
// sa_cell: plain __host__ __device__ code) thread by thread, phase by phase, with the shared-memory plane buffers in host
// memory, so that the tile logic (index maps, halos, k marching, carried faces, chunk seams) can be checked against the
// oracle without a GPU.  Built by tests/test_sa_emul.py with nvcc (host code only is executed).
#include <math.h>
#include <string.h>
#include <vector>
#include "../../adflow_b200/csrc/adfb_common.cuh"
#include "../../adflow_b200/csrc/sa_tile.cuh"

extern "C" {

struct SaEmulArrays {
    double *w, *rlv, *si, *sj, *sk, *vol, *volRef, *d2Wall, *dw;
    int32_t* iblank;
};

// the host chooser's tile (for the tests): out = TX, TY, kChunk, nT
int emul_sa_choose(int nx, int ny, int nz, int nPlanes, int nSM, int ctasPerSM, int* out) {
    const Dims d = make_dims(nx, ny, nz);
    const SaTile t = sa_tile_choose(d, nPlanes, nSM, ctasPerSM);
    out[0] = t.TX; out[1] = t.TY; out[2] = t.kChunk; out[3] = t.nT;
    return sa_tile_fits(t) ? 0 : 1;
}

// dw(itu1) of the planes 2+kOff .. min(kl, kTop); TX == 0: the chooser's tile on nSM multiprocessors with ctasPerSM CTAs each
int emul_sa(int nx, int ny, int nz, const AdfbParams* prm, const SaEmulArrays* a, int TX, int TY, int kChunk, int nSM, int ctasPerSM, int kOff,
            int kTop) {
    const Dims d = make_dims(nx, ny, nz);
    BlockDev b;
    memset(&b, 0, sizeof b);
    b.w = a->w; b.rlv = a->rlv; b.si = a->si; b.sj = a->sj; b.sk = a->sk; b.vol = a->vol; b.volRef = a->volRef; b.d2Wall = a->d2Wall;
    b.dw = a->dw; b.iblank = a->iblank;
    const AdfbParams& P = *prm;
    const double cb3Inv = 1.0 / P.rsaCb3, kar2Inv = 1.0 / (P.rsaK * P.rsaK);   // c_fheat[3], [4]
    const bool so = P.secondOrdTurb != 0;
    const int nPlanes = (kTop < d.kl ? kTop : d.kl) - (2 + kOff) + 1;
    if (nPlanes <= 0) return 0;
    const SaTile t = TX > 0 ? sa_tile_make(TX, TY, kChunk) : sa_tile_choose(d, nPlanes, nSM, ctasPerSM);
    if (!sa_tile_fits(t)) return 2;
    const int nbx = (d.nx + t.TX - 1) / t.TX, nby = (d.ny + t.TY - 1) / t.TY, nbz = (nPlanes + t.kChunk - 1) / t.kChunk;
    std::vector<double> smem(SA_NSLOT * SA_PLANE);
    std::vector<SaCtx> ctx(t.nT);
    std::vector<SaCarry> cr(t.nT);
    std::vector<SaOwn> own(t.nT), ownNext(t.nT);
    for (int bz = 0; bz < nbz; bz++)
        for (int by = 0; by < nby; by++)
            for (int bx = 0; bx < nbx; bx++) {
                // poison the shared buffers and the carry: anything read before it is written shows up as NaN
                for (double& v : smem) v = nan("");
                const int i0 = 2 + bx * t.TX, j0 = 2 + by * t.TY;
                const int ka = 2 + kOff + bz * t.kChunk;
                int kb = ka + t.kChunk - 1;
                if (kb > d.kl) kb = d.kl;
                if (kb > kTop) kb = kTop;
                auto slotBase = [&](int k) { return smem.data() + ((k - ka) % SA_NSLOT) * SA_PLANE; };
                auto slot = [&](int k) { return sa_plane(slotBase(k)); };
                // (the copies are plain stores here: a plane has landed as soon as it is loaded)
                for (int tid = 0; tid < t.nT; tid++) {
                    sa_load_plane(d, b, t, tid, i0, j0, ka, so, slot(ka));
                    sa_load_plane(d, b, t, tid, i0, j0, ka + 1, so, slot(ka + 1));
                    ctx[tid] = sa_ctx(d, t, tid, i0, j0);
                    double* p = reinterpret_cast<double*>(&cr[tid]);
                    for (size_t q = 0; q < sizeof(SaCarry) / sizeof(double); q++) p[q] = nan("");
                    sa_prologue(d, b, ctx[tid], ka, so, cr[tid]);
                    sa_own_loads(d, b, ctx[tid], ka, so, ownNext[tid]);
                    sa_finish_plane(d, t, tid, i0, j0, so, slot(ka));
                }
                for (int k = ka; k <= kb; k++) {
                    for (int tid = 0; tid < t.nT; tid++) {
                        if (k + 2 <= kb + 1) sa_load_plane(d, b, t, tid, i0, j0, k + 2, so, slot(k + 2));
                        own[tid] = ownNext[tid];
                        if (k < kb) sa_own_loads(d, b, ctx[tid], k + 1, so, ownNext[tid]);
                        sa_finish_plane(d, t, tid, i0, j0, so, slot(k + 1));
                    }
                    // (barrier)
                    for (int tid = 0; tid < t.nT; tid++) {
                        const SaCtx& x = ctx[tid];
                        if (!x.own) continue;
                        const double dwv = sa_cell(P, cb3Inv, kar2Inv, t, x, slot(k), slot(k + 1), own[tid], cr[tid]);
                        b.dw[5 * d.N + x.c0 + d.sK * k] = dwv;
                    }
                    // (barrier) plane k's buffer is free: poison it
                    for (int q = 0; q < SA_PLANE; q++) slotBase(k)[q] = nan("");
                }
            }
    return 0;
}

}  // extern "C"
