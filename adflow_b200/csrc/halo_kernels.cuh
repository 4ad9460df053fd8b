// halo_kernels.cuh -- device side of whalo1 / whalo2
// (src/utils/haloExchange.F90:5-199, whalo1to1RealGeneric :553-719)
//
// The reference packs `nVar` values per list entry into a host send buffer, posts
// MPI_Isend/Irecv per neighbour rank, copies same-rank donor->halo pairs directly and
// scatters the receive buffers.  Here the generic (block,i,j,k) index lists live on the
// device as (block, box offset) pairs; one gather kernel packs all neighbours' messages
// (SoA inside a message: value[var*count + entry], coalesced writes), NCCL moves them
// GPU to GPU over NVLink (grouped ncclSend/ncclRecv on the compute stream), one scatter
// kernel unpacks, one kernel does the same-rank copies.
#pragma once
#include "adfb_common.cuh"
#include <dlfcn.h>

#define ADFB_MAX_COMM_VARS 12

struct CommVarTable {
    // [block][var] -> device base pointer of that variable's box (nullptr beyond nVar)
    double* ptr[ADFB_MAX_COMM_VARS];
};

namespace {

// entries [0,n): gather var v of entry e into buf[msgBase[e's message] + v*msgCount + local e]
// message layout: message m (entries cum_m .. cum_m+count_m-1) starts at nVar*cum_m doubles;
// inside it value[v*count_m + local]
__global__ void __launch_bounds__(256) k_halo_pack(const int* __restrict__ entBlk, const long long* __restrict__ entOff,
                                                   const long long* __restrict__ entCum, const int* __restrict__ entLocal,
                                                   const int* __restrict__ entCount,
                                                   const CommVarTable* __restrict__ tab, int nVar, long long n,
                                                   double* __restrict__ buf) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n * nVar) return;
    const long long e = q % n;
    const int v = (int)(q / n);
    buf[(long long)nVar * entCum[e] + (long long)v * entCount[e] + entLocal[e]] = tab[entBlk[e]].ptr[v][entOff[e]];
}
__global__ void __launch_bounds__(256) k_halo_unpack(const int* __restrict__ entBlk, const long long* __restrict__ entOff,
                                                     const long long* __restrict__ entCum, const int* __restrict__ entLocal,
                                                     const int* __restrict__ entCount,
                                                     const CommVarTable* __restrict__ tab, int nVar, long long n,
                                                     const double* __restrict__ buf) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n * nVar) return;
    const long long e = q % n;
    const int v = (int)(q / n);
    tab[entBlk[e]].ptr[v][entOff[e]] = buf[(long long)nVar * entCum[e] + (long long)v * entCount[e] + entLocal[e]];
}
// overset donors (wOversetGeneric, haloExchange.F90:1471-1654): the value sent for a fringe cell is the weighted
// sum of the 8 cells (i..i+1, j..j+1, k..k+1) of the donor block, weights interp(1:8) in the reference's order
// (i fastest); sJ/sK of the donor block come with the entry
__device__ __forceinline__ double interp8(const double* __restrict__ v, long long o, long long sJ, long long sK,
                                          const double* __restrict__ w) {
    return w[0] * v[o] + w[1] * v[o + 1] + w[2] * v[o + sJ] + w[3] * v[o + 1 + sJ] + w[4] * v[o + sK] + w[5] * v[o + 1 + sK] +
           w[6] * v[o + sJ + sK] + w[7] * v[o + 1 + sJ + sK];
}
__global__ void __launch_bounds__(256) k_halo_pack_interp(const int* __restrict__ entBlk, const long long* __restrict__ entOff,
                                                          const long long* __restrict__ entCum, const int* __restrict__ entLocal,
                                                          const int* __restrict__ entCount, const long long* __restrict__ entSJ,
                                                          const long long* __restrict__ entSK, const double* __restrict__ wgt,
                                                          const CommVarTable* __restrict__ tab, int nVar, long long n,
                                                          double* __restrict__ buf) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n * nVar) return;
    const long long e = q % n;
    const int v = (int)(q / n);
    buf[(long long)nVar * entCum[e] + (long long)v * entCount[e] + entLocal[e]] =
        interp8(tab[entBlk[e]].ptr[v], entOff[e], entSJ[e], entSK[e], wgt + 8 * e);
}
__global__ void __launch_bounds__(256) k_halo_internal_interp(const int* __restrict__ srcBlk, const long long* __restrict__ srcOff,
                                                              const long long* __restrict__ srcSJ, const long long* __restrict__ srcSK,
                                                              const double* __restrict__ wgt, const int* __restrict__ dstBlk,
                                                              const long long* __restrict__ dstOff,
                                                              const CommVarTable* __restrict__ tab, int nVar, long long n) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n * nVar) return;
    const long long e = q % n;
    const int v = (int)(q / n);
    tab[dstBlk[e]].ptr[v][dstOff[e]] = interp8(tab[srcBlk[e]].ptr[v], srcOff[e], srcSJ[e], srcSK[e], wgt + 8 * e);
}
// same-rank donor -> halo copies (haloExchange.F90:654-676)
__global__ void __launch_bounds__(256) k_halo_internal(const int* __restrict__ srcBlk, const long long* __restrict__ srcOff,
                                                       const int* __restrict__ dstBlk, const long long* __restrict__ dstOff,
                                                       const CommVarTable* __restrict__ tab, int nVar, long long n) {
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n * nVar) return;
    const long long e = q % n;
    const int v = (int)(q / n);
    tab[dstBlk[e]].ptr[v][dstOff[e]] = tab[srcBlk[e]].ptr[v][srcOff[e]];
}


// orphanAverage (src/utils/haloExchange.F90:201-354): one thread per orphan.  A neighbour only counts when its iblank
// is 1 and an orphan's own iblank is not, so the orphans do not feed each other and the reference's sequential loop is
// order independent; the sums run over -i, +i, -j, +j, -k, +k like the reference's.
__global__ void __launch_bounds__(128) k_orphan_average(Dims d, BlockDev b, int nOrphans, const int32_t* __restrict__ orphans, int wStart, int wEnd,
                                                        int calcP, int calcLam, int calcEddy, double muInf, double eddyRatio) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= nOrphans) return;
    const int oi = orphans[3 * n], oj = orphans[3 * n + 1], ok = orphans[3 * n + 2];
    const long long N = d.N, c = ADFB_IDX(oi, oj, ok);
    double acc[9];
#pragma unroll
    for (int q = 0; q < 9; q++) acc[q] = 0.0;
    int nAvg = 0;
#pragma unroll
    for (int m = 0; m < 3; m++)
#pragma unroll
        for (int i = -1; i <= 1; i += 2) {
            const int ni = oi + (m == 0 ? i : 0), nj = oj + (m == 1 ? i : 0), nk = ok + (m == 2 ? i : 0);
            if (ni < 0 || ni > d.ib || nj < 0 || nj > d.jb || nk < 0 || nk > d.kb) continue;
            const long long cn = ADFB_IDX(ni, nj, nk);
            if (b.iblank[cn] != 1) continue;
            nAvg++;
            for (int l = wStart; l <= wEnd; l++) acc[l - 1] = acc[l - 1] + b.w[(l - 1) * N + cn];
            if (calcP) acc[6] = acc[6] + b.p[cn];
            if (calcLam) acc[7] = acc[7] + b.rlv[cn];
            if (calcEddy) acc[8] = acc[8] + b.rev[cn];
        }
    if (nAvg > 0) {
        const double r = (double)nAvg;
        for (int l = wStart; l <= wEnd; l++) b.w[(l - 1) * N + c] = acc[l - 1] / r;
        if (calcP) b.p[c] = acc[6] / r;
        if (calcLam) b.rlv[c] = acc[7] / r;
        if (calcEddy) b.rev[c] = acc[8] / r;
    } else {
        for (int l = wStart; l <= wEnd; l++) b.w[(l - 1) * N + c] = c_prm.wInf[l - 1];
        if (calcP) b.p[c] = c_prm.pInfCorr;
        if (calcLam) b.rlv[c] = muInf;
        if (calcEddy) b.rev[c] = eddyRatio * muInf;
    }
}

}  // namespace

// ---------------------------------------------------------------------------
// NCCL, resolved at run time (dlopen) so that the library also loads where no NCCL is
// installed; only multi-rank runs need it.
typedef struct ncclComm* ncclComm_t_;
struct Id128 { char b[128]; };  // ncclUniqueId is passed BY VALUE to ncclCommInitRank
struct NcclApi {
    void* h = nullptr;
    int (*GetUniqueId)(void*) = nullptr;
    int (*CommInitRank)(ncclComm_t_*, int, Id128, int) = nullptr;
    int (*CommDestroy)(ncclComm_t_) = nullptr;
    int (*Send)(const void*, size_t, int, int, ncclComm_t_, cudaStream_t) = nullptr;
    int (*Recv)(void*, size_t, int, int, ncclComm_t_, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, ncclComm_t_, cudaStream_t) = nullptr;
    int (*GroupStart)() = nullptr;
    int (*GroupEnd)() = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool load(std::string& err) {
        if (h) return true;
        const char* names[] = {"libnccl.so.2", "libnccl.so"};
        for (const char* n : names) { h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); if (h) break; }
        if (!h) { err = std::string("cannot dlopen libnccl.so.2: ") + dlerror(); return false; }
#define ADFB_SYM(field, name) *(void**)(&field) = dlsym(h, name); if (!field) { err = std::string("missing NCCL symbol ") + name; return false; }
        ADFB_SYM(GetUniqueId, "ncclGetUniqueId");
        ADFB_SYM(CommInitRank, "ncclCommInitRank");
        ADFB_SYM(CommDestroy, "ncclCommDestroy");
        ADFB_SYM(Send, "ncclSend");
        ADFB_SYM(Recv, "ncclRecv");
        ADFB_SYM(AllReduce, "ncclAllReduce");
        ADFB_SYM(GroupStart, "ncclGroupStart");
        ADFB_SYM(GroupEnd, "ncclGroupEnd");
        ADFB_SYM(GetErrorString, "ncclGetErrorString");
#undef ADFB_SYM
        return true;
    }
};
static const int kNcclDouble = 8;  // ncclFloat64 (nccl.h ncclDataType_t)
static const int kNcclSum = 0;     // ncclSum
static const int kNcclMax = 2;     // ncclMax
static const int kNcclMin = 3;     // ncclMin (nccl.h ncclRedOp_t: sum, prod, max, min)
