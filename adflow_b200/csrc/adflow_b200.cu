// adflow_b200.cu -- C ABI of libadflow_b200.so (include/adflow_b200.h) and the
// host-side block registry.  Single translation unit: the kernel families are
// implementation headers (*_kernels.cuh) so that the constant-memory parameter
// block is shared without relocatable device code.
//
// There is no CPU fallback anywhere in this file: every entry point needs a
// live CUDA context and fails with a message otherwise.
#include <cuda_runtime.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>

#include <map>
#include <string>
#include <vector>
#include <algorithm>

#include "adfb_common.cuh"
#include "state_kernels.cuh"
#include "residual_kernels.cuh"
#include "smoother_kernels.cuh"
#include "mg_kernels.cuh"
#include "ank_kernels.cuh"
#include "krylov_kernels.cuh"
#include "halo_kernels.cuh"
#include "dadi_kernels.cuh"
#include "sa_kernels.cuh"

namespace {

struct Block {
    bool alive = false;
    int level = 1, nw = 6, rightHanded = 1;
    Dims d;
    BlockDev dev;
    std::vector<void*> allocs;
    bool haveMetrics = false;
    std::vector<AdfbSubface> subfaces;  // host copies (device arrays in bcDev)
    std::vector<void*> bcAllocs;
    // multigrid: the next finer / coarser block of the same mesh block and the transfer tables (on the coarse
    // block: mg?Fine, mg?Weight; the fine block's mg?Coarse are kept with the coarse block as well)
    int fineBlk = -1, coarseBlk = -1;
    MgTables mg = {};
    // overset orphans (blockPointers nOrphans / orphans) and the free-stream viscosities orphanAverage falls back to
    int nOrphans = 0;
    int32_t* dOrphans = nullptr;
    double muInf = 0.0, eddyVisInfRatio = 0.0;
    std::vector<void*> mgAllocs;
};

struct Context {
    bool ready = false;
    int device = -1, rank = 0, nranks = 1;
    cudaStream_t stream = nullptr;
    LaunchEnv env;
    // halo exchange split around the BCs (multi-rank): pack and send / receive run on commStream
    cudaStream_t commStream = nullptr;
    cudaEvent_t evPost = nullptr, evDone = nullptr;
    // slab pipeline of the form function: copies in, copies out, back end of a slab; [0..2][slab] and [3][fork / join]
    cudaStream_t ffIn = nullptr, ffOut = nullptr, ffBack = nullptr;
    cudaEvent_t ffEv[4][34] = {};
    double* dConst = nullptr;   // parameter constants formed on the device (adfb_set_params)
    AdfbParams prm;
    bool havePrm = false;
    std::vector<Block> blocks;
    double* dRed = nullptr;   // reduction scratch
    size_t dRedN = 0;
    double* hRed = nullptr;   // pinned
    double* dVec = nullptr;   // AoS staging vector (get/set states, get res)
    size_t dVecN = 0;
    // NK / MFFD device vectors: direction a, base state U, base residual F(U), result y
    double *nkA = nullptr, *nkU = nullptr, *nkF0 = nullptr, *nkY = nullptr;
    size_t nkN = 0;
    bool nkHaveBase = false;
    double nkUnorm = 0.0, nkLastH = 0.0;
    MffdDev* dMffd = nullptr;     // record of the fused matrix-free product (device) and its pinned host image
    MffdDev* hMffd = nullptr;
    bool mffdFuse = false;        // adfb_residual: skip k_state_prep (done by k_nkvec_prep) and form y in the kernels that write dw
    std::string err;
    // multi-rank
    NcclApi nccl;
    ncclComm_t_ comm = nullptr;
    // 1-to-1 communication pattern (commPatternCell_2nd + internalCell_2nd,
    // src/modules/communication.F90:85-168), device resident
    struct Pattern {
        bool set = false;
        std::vector<int> nbrRank, sendCount, recvCount;
        long long nSend = 0, nRecv = 0, nInt = 0;
        int *sBlk = nullptr, *sLocal = nullptr, *sCount = nullptr; long long *sOff = nullptr, *sCum = nullptr;
        int *rBlk = nullptr, *rLocal = nullptr, *rCount = nullptr; long long *rOff = nullptr, *rCum = nullptr;
        int *iSrcBlk = nullptr, *iDstBlk = nullptr; long long *iSrcOff = nullptr, *iDstOff = nullptr;
        double *sendBuf = nullptr, *recvBuf = nullptr;
        // overset pattern only: donor-block strides and the 8 interpolation weights per send / internal entry
        bool interp = false;
        long long *sSJ = nullptr, *sSK = nullptr, *iSJ = nullptr, *iSK = nullptr;
        double *sW = nullptr, *iW = nullptr;
        CommVarTable* dTab = nullptr;   // unused (kept for layout); tables are cached per selection
        int tabBlocks = 0;
        std::map<int, CommVarTable*> tabs;  // key: start | end<<4 | commP<<8 | commV<<9
        std::vector<void*> allocs;
    };
    // per grid level: 1-to-1 (commPatternCell_2nd / internalCell_2nd; _1st lists on coarse levels) and overset
    // (commPatternOverset / internalOverset)
    std::map<int, Pattern> pats, ovPats;
    // CUDA graphs of whole entry points (launch-latency bound sequences of small kernels)
    std::map<unsigned long long, cudaGraphExec_t> graphs;
    std::map<unsigned long long, long long> graphLaunches;
    std::vector<unsigned long long> ffKeys;   // graphs of the pipelined form function, oldest first (at most 8 kept)
    bool useGraphs = true;
    bool capturing = false;
    // ANK (module ANKSolver): options, per-cell time-step blocks, the perturbed vector of the last product
    AdfbAnkParams ank;
    bool haveAnk = false, ankHaveT = false, ankHaveBase = false, ankTurbHaveBase = false;
    double *ankT = nullptr, *ankPert = nullptr;
    size_t ankTN = 0, ankPertN = 0;
    double ankUnorm = 0.0;
    // device GMRES workspace: (restart + 2) vectors + reduction scratch
    double *kryV = nullptr, *kryRed = nullptr;
    size_t kryVN = 0;
    int mgInitWr = 1;   // coarse-level smoother residual starts from wr (0 inside transferToCoarseGrid: from zero)
    int groundLevel = 1;   // iteration%groundLevel: the finest level of the current multigrid cycle (> 1 during the full-multigrid start-up)
};

Context g;

// currentLevel > groundLevel: the coarse-level branches of the smoother path (dw = wr start, first-order dissipation, first
// halos only, frozen eddy viscosity, constant-pressure walls); levels <= groundLevel run the fine-grid routines.
static inline bool above_ground(int level) { return level > g.groundLevel; }
// The discretisation of a residual on `level`.  The blockette path (blocketteRes: adfb_residual, the form function, the
// matrix-free products, ANK) selects spaceDiscr on every level (blockette.F90:637-653); the block path of the smoothers and
// of multigrid (residual_block) selects spaceDiscrCoarse unless currentLevel == 1 (residuals.F90:71-75).  So a coarse ground
// level of the full-multigrid start-up runs its first smoothing step on a residual of the fine discretisation (solveState's
// computeResidualNK, solvers.F90:1014-1018) and every later one on the fine-grid routines of the coarse discretisation.
static inline int residual_discr(int level, bool blockette) {
    return (blockette || level == 1) ? g.prm.spaceDiscr : g.prm.spaceDiscrCoarse;
}

int fail(const char* fmt, ...) {
    char buf[1024];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    g.err = buf;
    return 1;
}

#define CK(call)                                                                                      \
    do {                                                                                              \
        cudaError_t e_ = (call);                                                                      \
        if (e_ != cudaSuccess) return fail("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); \
    } while (0)

#define NEED_INIT()                                                      \
    do {                                                                 \
        if (!g.ready) return fail("adfb_init has not been called (no CUDA device bound)"); \
    } while (0)

Block* get_block(int blk) {
    if (blk < 0 || blk >= (int)g.blocks.size() || !g.blocks[blk].alive) return nullptr;
    return &g.blocks[blk];
}

template <typename T>
int dalloc(Block& b, T** p, size_t n) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T));
    if (e != cudaSuccess) return fail("cudaMalloc(%zu bytes): %s", n * sizeof(T), cudaGetErrorString(e));
    e = cudaMemsetAsync(q, 0, n * sizeof(T), g.stream);
    if (e != cudaSuccess) return fail("cudaMemset: %s", cudaGetErrorString(e));
    b.allocs.push_back(q);
    *p = (T*)q;
    return 0;
}

// Copy a host Fortran array with reference extents lo:lo+n-1 (per dimension) and
// ncomp trailing components into / out of the uniform device box.
int copy_box(const Dims& d, void* dev, const void* host, const int lo[3], const int n[3], int ncomp, size_t es,
             bool toDevice) {
    const bool full = lo[0] == 0 && lo[1] == 0 && lo[2] == 0 && n[0] == d.NI && n[1] == d.NJ && n[2] == d.NK;
    if (full) {
        const size_t bytes = (size_t)d.N * ncomp * es;
        if (toDevice) CK(cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, g.stream));
        else CK(cudaMemcpyAsync((void*)host, dev, bytes, cudaMemcpyDeviceToHost, g.stream));
        return 0;
    }
    const size_t hostComp = (size_t)n[0] * n[1] * n[2] * es;
    for (int m = 0; m < ncomp; m++) {
        cudaMemcpy3DParms p;
        memset(&p, 0, sizeof p);
        cudaPitchedPtr hp = make_cudaPitchedPtr((char*)host + m * hostComp, n[0] * es, n[0] * es, n[1]);
        cudaPitchedPtr dp = make_cudaPitchedPtr((char*)dev + (size_t)m * d.N * es, d.NI * es, d.NI * es, d.NJ);
        p.extent = make_cudaExtent(n[0] * es, n[1], n[2]);
        if (toDevice) {
            p.srcPtr = hp; p.dstPtr = dp;
            p.dstPos = make_cudaPos(lo[0] * es, lo[1], lo[2]);
            p.kind = cudaMemcpyHostToDevice;
        } else {
            p.srcPtr = dp; p.dstPtr = hp;
            p.srcPos = make_cudaPos(lo[0] * es, lo[1], lo[2]);
            p.kind = cudaMemcpyDeviceToHost;
        }
        CK(cudaMemcpy3DAsync(&p, g.stream));
    }
    return 0;
}

enum Ext { C2, C1, C0, NODE, FI, FJ, FK, PI_, PJ_, PK_ };
void extents(const Dims& d, Ext e, int lo[3], int n[3]) {
    switch (e) {
        case C2: lo[0] = lo[1] = lo[2] = 0; n[0] = d.NI; n[1] = d.NJ; n[2] = d.NK; break;
        case C1: lo[0] = lo[1] = lo[2] = 1; n[0] = d.ie; n[1] = d.je; n[2] = d.ke; break;
        case C0: lo[0] = lo[1] = lo[2] = 2; n[0] = d.nx; n[1] = d.ny; n[2] = d.nz; break;
        case NODE: lo[0] = lo[1] = lo[2] = 0; n[0] = d.ie + 1; n[1] = d.je + 1; n[2] = d.ke + 1; break;
        case FI: lo[0] = 0; lo[1] = 1; lo[2] = 1; n[0] = d.ie + 1; n[1] = d.je; n[2] = d.ke; break;
        case FJ: lo[0] = 1; lo[1] = 0; lo[2] = 1; n[0] = d.ie; n[1] = d.je + 1; n[2] = d.ke; break;
        case FK: lo[0] = 1; lo[1] = 1; lo[2] = 0; n[0] = d.ie; n[1] = d.je; n[2] = d.ke + 1; break;
        case PI_: lo[0] = 1; lo[1] = 2; lo[2] = 2; n[0] = d.il; n[1] = d.ny; n[2] = d.nz; break;
        case PJ_: lo[0] = 2; lo[1] = 1; lo[2] = 2; n[0] = d.nx; n[1] = d.jl; n[2] = d.nz; break;
        case PK_: lo[0] = 2; lo[1] = 2; lo[2] = 1; n[0] = d.nx; n[1] = d.ny; n[2] = d.kl; break;
    }
}
int put(const Block& b, Ext e, void* dev, const void* host, int ncomp, size_t es) {
    int lo[3], n[3];
    extents(b.d, e, lo, n);
    return copy_box(b.d, dev, host, lo, n, ncomp, es, true);
}
int get(const Block& b, Ext e, const void* dev, void* host, int ncomp, size_t es) {
    int lo[3], n[3];
    extents(b.d, e, lo, n);
    return copy_box(b.d, (void*)dev, host, lo, n, ncomp, es, false);
}

// Run `body` through a cached CUDA graph: the entry points are sequences of 10-25 small
// kernels (BC subfaces, halo pack/unpack ...) whose launch latency would otherwise dominate.
// Graphs are bypassed while per-kernel event timing is on (and for multi-rank runs when
// ADFB_GRAPH_NCCL=0 disables capturing NCCL send/recv).
template <typename F>
int run_graphed(unsigned long long key, F body) {
    static int ncclOk = -1;
    if (ncclOk < 0) {
        const char* e = getenv("ADFB_GRAPH_NCCL"); ncclOk = (e && e[0] == '0') ? 0 : 1;  // NCCL send/recv capture fine with NCCL >= 2.9
        const char* n = getenv("ADFB_NO_GRAPH"); if (n && n[0] == '1') g.useGraphs = false;
    }
    // an entry point called from inside another one's capture runs inline (the flag lives in the context: a
    // function-local static would be one per template instantiation)
    if (!g.useGraphs || g_kt.on || g.capturing || (g.nranks > 1 && !ncclOk)) return body();
    auto it = g.graphs.find(key);
    if (it == g.graphs.end()) {
        // relaxed mode: the lazily built halo variable tables may cudaMalloc/cudaMemcpy (on the
        // legacy stream, which does not synchronise with the non-blocking compute stream)
        cudaGraph_t graph = nullptr;
        CK(cudaStreamBeginCapture(g.stream, cudaStreamCaptureModeRelaxed));
        const long long l0 = g_kt.launches;
        g.capturing = true;
        const int rc = body();
        g.capturing = false;
        const long long nl = g_kt.launches - l0;
        cudaError_t e = cudaStreamEndCapture(g.stream, &graph);
        if (rc != 0) {   // the entry point itself failed (misuse): report it; graphs stay enabled for later calls
            if (graph) cudaGraphDestroy(graph);
            cudaGetLastError();
            return rc;
        }
        if (e != cudaSuccess || !graph) {
            if (graph) cudaGraphDestroy(graph);
            cudaGetLastError();
            g.useGraphs = false;  // capture is not possible here: direct launches for the rest of the run
            return body();
        }
        cudaGraphExec_t exec = nullptr;
        e = cudaGraphInstantiate(&exec, graph, 0);
        cudaGraphDestroy(graph);
        if (e != cudaSuccess) { g.useGraphs = false; cudaGetLastError(); return body(); }
        g.graphs[key] = exec;
        g.graphLaunches[key] = nl;
        it = g.graphs.find(key);
    }
    CK(cudaGraphLaunch(it->second, g.stream));
    g_kt.launches += g.graphLaunches[key];
    return 0;
}
// the cached per-pattern variable tables hold raw block pointers and the variable selection of the equation set:
// they go whenever blocks or parameters change (the allocations stay with the pattern until it is reset)
void drop_comm_tables() {
    for (auto* m : {&g.pats, &g.ovPats})
        for (auto& kv : *m) kv.second.tabs.clear();
}
void drop_graphs() {
    drop_comm_tables();
    for (auto& kv : g.graphs) cudaGraphExecDestroy(kv.second);
    g.graphs.clear();
    g.graphLaunches.clear();
    g.ffKeys.clear();
}

// The streams, events and buffers of the context, for the device that is current.  The library stream carries the
// latency-bound chains (BC levels, line solves) at the highest priority, and so does the stream of the SA row forked beside
// the flow rows: that is the priority the SA row has run and been measured at (cudaStreamCopyAttributes from the library
// stream, which carries the priority attribute, used to precede every fork).
int create_device_resources() {
    int prLo = 0, prHi = 0;
    CK(cudaDeviceGetStreamPriorityRange(&prLo, &prHi));
    for (cudaStream_t* s : {&g.stream, &g.env.saStream}) CK(cudaStreamCreateWithPriority(s, cudaStreamNonBlocking, prHi));
    for (cudaStream_t* s : {&g.commStream, &g.ffIn, &g.ffOut, &g.ffBack}) CK(cudaStreamCreateWithFlags(s, cudaStreamNonBlocking));
    for (cudaEvent_t* e : {&g.env.saFork, &g.env.saJoin, &g.evPost, &g.evDone}) CK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    for (auto& row : g.ffEv) for (cudaEvent_t& e : row) CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    CK(cudaMalloc((void**)&g.dConst, 8 * sizeof(double)));
    CK(cudaMallocHost((void**)&g.hRed, 256 * sizeof(double)));
    return 0;
}
void release_device_resources() {
    for (cudaEvent_t* e : {&g.env.saFork, &g.env.saJoin, &g.evPost, &g.evDone}) { if (*e) cudaEventDestroy(*e); *e = nullptr; }
    for (auto& row : g.ffEv) for (cudaEvent_t& e : row) { if (e) cudaEventDestroy(e); e = nullptr; }
    for (cudaStream_t* s : {&g.stream, &g.env.saStream, &g.commStream, &g.ffIn, &g.ffOut, &g.ffBack}) { if (*s) cudaStreamDestroy(*s); *s = nullptr; }
    if (g.dConst) cudaFree(g.dConst);
    g.dConst = nullptr;
    if (g.hRed) cudaFreeHost(g.hRed);
    g.hRed = nullptr;
}

}  // namespace

// ===========================================================================
extern "C" {

int adfb_last_error(char* buf, int n) {
    if (!buf || n <= 0) return 1;
    snprintf(buf, n, "%s", g.err.c_str());
    return 0;
}

int adfb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
    return n;
}

int adfb_get_unique_id(void* out128) {
    if (!out128) return fail("adfb_get_unique_id: null buffer");
    std::string e;
    if (!g.nccl.load(e)) return fail("adfb_get_unique_id: %s", e.c_str());
    const int rc = g.nccl.GetUniqueId(out128);
    if (rc != 0) return fail("ncclGetUniqueId: %s", g.nccl.GetErrorString(rc));
    return 0;
}

int adfb_init(int device, const void* ncclUniqueId, int rank, int nranks) {
    (void)ncclUniqueId;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail("adfb_init: no CUDA device available (%s); this library has no CPU path",
                    e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    if (device < 0 || device >= n) return fail("adfb_init: device %d out of range (0..%d)", device, n - 1);
    // the streams, events and buffers belong to the device they were created on
    if (g.stream && device != g.device)
        return fail("adfb_init: the context is bound to device %d; adfb_finalize it before binding device %d", g.device, device);
    CK(cudaSetDevice(device));
    if (!g.stream) {
        if (create_device_resources()) {
            release_device_resources();
            return 1;
        }
        g.device = device;
    }
    {
        int v = 0;
        CK(cudaDeviceGetAttribute(&g.env.nSM, cudaDevAttrMultiProcessorCount, device));
        CK(cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
        g.env.smemOptin = (size_t)v;
        // the kernels that take more dynamic shared memory than the default 48 KiB
        for (const void* k : {(const void*)k_flowres<true, true>, (const void*)k_flowres<true, false>, (const void*)k_flowres<false, true>,
                              (const void*)k_flowres<false, false>})
            CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, v));
        CK(cudaFuncSetAttribute(k_resavg_lines, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kResavgSmemMax));
        CK(cudaFuncSetAttribute(k_dadi_thomas_tile, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kDadiTileSmem));
    }
    g.device = device; g.rank = rank; g.nranks = nranks;
    g.err.clear();
    if (g.comm) { g.nccl.CommDestroy(g.comm); g.comm = nullptr; }   // re-init: the previous communicator goes
    if (nranks > 1) {
        g.ready = false; g.nranks = 1;   // a failing NCCL set-up must not leave a multi-rank context without a communicator
        if (!ncclUniqueId) return fail("adfb_init: nranks > 1 needs the 128-byte NCCL unique id of rank 0");
        std::string e;
        if (!g.nccl.load(e)) return fail("adfb_init: %s", e.c_str());
        Id128 id;
        memcpy(id.b, ncclUniqueId, 128);
        const int rc = g.nccl.CommInitRank(&g.comm, nranks, id, rank);
        if (rc != 0) { g.comm = nullptr; return fail("ncclCommInitRank: %s", g.nccl.GetErrorString(rc)); }
        g.nranks = nranks;
    }
    g.ready = true;
    return 0;
}

int adfb_finalize(void) {
    if (!g.ready) return 0;
    // the graphs first: the pipelined form function's graphs hold the context's events
    drop_graphs();
    cudaStreamSynchronize(g.stream);
    for (size_t i = 0; i < g.blocks.size(); i++)
        if (g.blocks[i].alive) adfb_block_destroy((int)i);
    g.blocks.clear();
    if (g.dRed) cudaFree(g.dRed);
    g.dRed = nullptr; g.dRedN = 0;
    if (g.dMffd) { cudaFree(g.dMffd); g.dMffd = nullptr; }
    if (g.hMffd) { cudaFreeHost(g.hMffd); g.hMffd = nullptr; }
    if (g.dVec) cudaFree(g.dVec);
    g.dVec = nullptr; g.dVecN = 0;
    for (double** p : {&g.nkA, &g.nkU, &g.nkF0, &g.nkY}) { if (*p) cudaFree(*p); *p = nullptr; }
    g.nkN = 0;
    g.nkHaveBase = false; g.ankHaveBase = false; g.ankTurbHaveBase = false;   // the base vectors went with the buffers g.nkHaveBase = false;
    // ANK / Krylov state belongs to the context as well: a later adfb_init starts from scratch
    for (double** p : {&g.ankT, &g.ankPert, &g.kryV, &g.kryRed}) { if (*p) cudaFree(*p); *p = nullptr; }
    g.ankTN = 0; g.ankPertN = 0; g.kryVN = 0;
    g.haveAnk = false; g.ankHaveT = false; g.ankHaveBase = false;
    // so do the parameters and the multigrid position: a later context starts on ground level 1 and must set its parameters
    g.havePrm = false;
    g.groundLevel = 1; g.mgInitWr = 1;
    for (auto* M : {&g.pats, &g.ovPats}) {
        for (auto& kv : *M) for (void* q : kv.second.allocs) cudaFree(q);
        M->clear();
    }
    if (g.comm) { g.nccl.CommDestroy(g.comm); g.comm = nullptr; }
    release_device_resources();
    g_kt.collect();
    for (cudaEvent_t e : g_kt.pool) cudaEventDestroy(e);
    g_kt.pool.clear();
    g.ready = false;
    return 0;
}

int adfb_synchronize(void) {
    NEED_INIT();
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

long long adfb_launch_count(void) { return g_kt.launches; }
int adfb_graph_count(void) { return g.useGraphs ? (int)g.graphs.size() : -1; }
/* per-kernel CUDA-event timing (bench.py roofline pass): on=1 starts recording and
   resets the accumulators; adfb_kernel_times synchronises and returns the
   cumulative milliseconds and launch counts per kernel family. */
int adfb_set_timing(int on) {
    NEED_INIT();
    CK(cudaStreamSynchronize(g.stream));
    g_kt.reset();
    g_kt.on = on != 0;
    return 0;
}
int adfb_kernel_times(double* ms, long long* counts, int n) {
    NEED_INIT();
    CK(cudaStreamSynchronize(g.stream));
    g_kt.collect();
    for (int i = 0; i < n && i < K_NUM; i++) { ms[i] = g_kt.ms[i]; counts[i] = g_kt.count[i]; }
    return K_NUM;
}
const char* adfb_kernel_name(int id) { return (id >= 0 && id < K_NUM) ? kKernelNames[id] : ""; }
void* adfb_stream(void) { return (void*)g.stream; }

int adfb_set_params(const AdfbParams* prm) {
    NEED_INIT();
    drop_graphs();
    if (!prm) return fail("adfb_set_params: null");
    if (prm->equations < ADFB_EULER || prm->equations > ADFB_RANS) return fail("adfb_set_params: bad equations %d", prm->equations);
    if (prm->spaceDiscr != ADFB_DISS_SCALAR && prm->spaceDiscr != ADFB_DISS_MATRIX && prm->spaceDiscr != ADFB_UPWIND)
        return fail("adfb_set_params: unknown spaceDiscr %d", prm->spaceDiscr);
    if (prm->spaceDiscrCoarse != ADFB_DISS_SCALAR && prm->spaceDiscrCoarse != ADFB_DISS_MATRIX && prm->spaceDiscrCoarse != ADFB_UPWIND)
        return fail("adfb_set_params: unknown spaceDiscrCoarse %d", prm->spaceDiscrCoarse);
    if (prm->useRotationSA && prm->turbProd == ADFB_PROD_VORTICITY)
        return fail("adfb_set_params: useRotationSA with vorticity production reads an unset strainMag2 in the "
                    "reference (src/turbulence/sa.F90:273); unsupported");
    g.prm = *prm;
    g.havePrm = true;
    CK(cudaMemcpyToSymbolAsync(c_prm, &g.prm, sizeof(AdfbParams), 0, cudaMemcpyHostToDevice, g.stream));
    {
        double fheat[16] = {};
        const double gm1 = g.prm.gammaInf - 1.0;
        fheat[0] = 1.0 / (g.prm.prandtl * gm1); fheat[1] = 1.0 / (g.prm.prandtlTurb * gm1);
        fheat[3] = 1.0 / g.prm.rsaCb3; fheat[4] = 1.0 / (g.prm.rsaK * g.prm.rsaK);
        fheat[7] = 1.0 / gm1; fheat[8] = 0.000001 * g.prm.gammaInf * g.prm.pInfCorr / g.prm.rhoInf;
        CK(cudaMemcpyToSymbolAsync(c_fheat, fheat, sizeof fheat, 0, cudaMemcpyHostToDevice, g.stream));
        k_param_consts<<<1, 1, 0, g.stream>>>(g.dConst);   // reads the c_prm uploaded above (stream order)
        CK(cudaMemcpyToSymbolAsync(c_fheat, g.dConst, sizeof(double), 2 * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
        CK(cudaMemcpyToSymbolAsync(c_fheat, g.dConst + 1, 2 * sizeof(double), 5 * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
        CK(cudaStreamSynchronize(g.stream));
    }
    {
        static int trig = -1;
        if (trig < 0) { const char* e = getenv("ADFB_PDL_TRIGGER"); trig = e ? atoi(e) : 0; }
        CK(cudaMemcpyToSymbolAsync(c_pdlTrigger, &trig, sizeof(int), 0, cudaMemcpyHostToDevice, g.stream));
    }
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

int adfb_block_create(int blk, int level, int nx, int ny, int nz, int nw, int rightHanded) {
    NEED_INIT();
    drop_graphs();
    if (blk < 0 || blk > 4095) return fail("adfb_block_create: block id %d out of range", blk);
    if (nx < 1 || ny < 1 || nz < 1) return fail("adfb_block_create: bad extents %d %d %d", nx, ny, nz);
    if (nw != 5 && nw != 6) return fail("adfb_block_create: nw must be 5 (Euler/NS) or 6 (RANS-SA), got %d", nw);
    if ((int)g.blocks.size() <= blk) g.blocks.resize(blk + 1);
    if (g.blocks[blk].alive) return fail("adfb_block_create: block %d already exists", blk);
    Block& b = g.blocks[blk];
    b = Block();
    b.level = level; b.nw = nw; b.rightHanded = rightHanded;
    b.d = make_dims(nx, ny, nz);
    const size_t N = (size_t)b.d.N;
    BlockDev& v = b.dev;
    memset(&v, 0, sizeof v);
    int rc = 0;
    // state slab: w(nw), p, rlv, rev contiguous (the tile kernel loads it through one tensor map)
    rc |= dalloc(b, &v.w, N * (nw + 3));
    v.p = v.w + N * nw; v.rlv = v.p + N; v.rev = v.rlv + N;
    rc |= dalloc(b, &v.x, N * 3); rc |= dalloc(b, &v.si, N * 3); rc |= dalloc(b, &v.sj, N * 3); rc |= dalloc(b, &v.sk, N * 3);
    rc |= dalloc(b, &v.vol, N); rc |= dalloc(b, &v.volRef, N); rc |= dalloc(b, &v.d2Wall, N);
    rc |= dalloc(b, &v.porI, N); rc |= dalloc(b, &v.porJ, N); rc |= dalloc(b, &v.porK, N); rc |= dalloc(b, &v.iblank, N);
    rc |= dalloc(b, &v.dw, N * nw); rc |= dalloc(b, &v.fw, N * 5);
    rc |= dalloc(b, &v.ss, N); rc |= dalloc(b, &v.dss, N * 3);
    rc |= dalloc(b, &v.aa, N); rc |= dalloc(b, &v.radI, N); rc |= dalloc(b, &v.radJ, N); rc |= dalloc(b, &v.radK, N);
    rc |= dalloc(b, &v.dtl, N); rc |= dalloc(b, &v.grad, N * 12);
    rc |= dalloc(b, &v.wn, N * 5); rc |= dalloc(b, &v.pn, N); rc |= dalloc(b, &v.scratch, N * 10);
    rc |= dalloc(b, &v.ssum, N * 9); rc |= dalloc(b, &v.sv, N * 9); rc |= dalloc(b, &v.ovol, N);
    rc |= dalloc(b, &v.vn, N * 12); rc |= dalloc(b, &v.flux, N * 30); rc |= dalloc(b, &v.shock, N);
    rc |= dalloc(b, &v.wr, N * 5); rc |= dalloc(b, &v.w1, N * 5); rc |= dalloc(b, &v.p1, N);
    v.coarse = level > 1 ? 1 : 0;
    {
        const long long pI = (long long)b.d.NJ * b.d.NK, pJ = (long long)b.d.NI * b.d.NK, pK = (long long)b.d.NI * b.d.NJ;
        v.wallP = pI > pJ ? (pI > pK ? pI : pK) : (pJ > pK ? pJ : pK);
        rc |= dalloc(b, &v.wallTau, (size_t)(3 * 2 * 9) * v.wallP);
    }
    if (rc) {
        for (void* q : b.allocs) cudaFree(q);
        b.allocs.clear();
        return 1;
    }
    b.alive = true;
    return 0;
}

int adfb_block_destroy(int blk) {
    NEED_INIT();
    drop_graphs();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_block_destroy: no block %d", blk);
    cudaStreamSynchronize(g.stream);
    for (void* q : b->allocs) cudaFree(q);
    for (void* q : b->bcAllocs) cudaFree(q);
    for (void* q : b->mgAllocs) cudaFree(q);
    if (b->dOrphans) cudaFree(b->dOrphans);
    *b = Block();
    return 0;
}

int adfb_block_set_geometry(int blk, const double* x, const double* si, const double* sj, const double* sk,
                            const double* vol, const double* volRef, const double* d2Wall, const int8_t* porI,
                            const int8_t* porJ, const int8_t* porK, const int32_t* iblank) {
    NEED_INIT();
    // No drop_graphs: a mesh warp rewrites the block's geometry arrays in place, and the cached graphs hold only their
    // addresses and the block extents, which do not change (the same holds for the state uploads).
    Block* b = get_block(blk);
    if (!b) return fail("adfb_block_set_geometry: no block %d", blk);
    if (!x || !vol || !volRef || !porI || !porJ || !porK || !iblank)
        return fail("adfb_block_set_geometry: x, vol, volRef, porI/J/K and iblank are required");
    if (b->nw > 5 && !d2Wall) return fail("adfb_block_set_geometry: d2Wall is required for RANS blocks");
    const BlockDev& v = b->dev;
    if (put(*b, NODE, v.x, x, 3, 8)) return 1;
    if (si && sj && sk) {
        if (put(*b, FI, v.si, si, 3, 8) || put(*b, FJ, v.sj, sj, 3, 8) || put(*b, FK, v.sk, sk, 3, 8)) return 1;
    } else if (si || sj || sk) {
        return fail("adfb_block_set_geometry: pass all of si, sj, sk or none");
    } else {
        if (launch_metrics(b->d, v, b->rightHanded, g.stream)) return fail("metrics kernel launch failed");
    }
    if (put(*b, C2, v.vol, vol, 1, 8) || put(*b, C2, v.volRef, volRef, 1, 8)) return 1;
    if (d2Wall && put(*b, C0, v.d2Wall, d2Wall, 1, 8)) return 1;
    if (put(*b, PI_, v.porI, porI, 1, 1) || put(*b, PJ_, v.porJ, porJ, 1, 1) || put(*b, PK_, v.porK, porK, 1, 1)) return 1;
    if (put(*b, C2, v.iblank, iblank, 1, 4)) return 1;
    if (launch_geom(b->d, v, g.stream)) return fail("geometry kernel launch failed");
    CK(cudaStreamSynchronize(g.stream));
    b->haveMetrics = true;
    return 0;
}

int adfb_block_set_bc(int blk, int nSub, const AdfbSubface* subfaces) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_block_set_bc: no block %d", blk);
    drop_graphs();
    if (nSub < 0 || (nSub > 0 && !subfaces)) return fail("adfb_block_set_bc: bad arguments");
    cudaStreamSynchronize(g.stream);
    for (void* q : b->bcAllocs) cudaFree(q);
    b->bcAllocs.clear();
    b->subfaces.clear();
    for (int s = 0; s < nSub; s++) {
        AdfbSubface sf = subfaces[s];
        if (sf.faceId < ADFB_IMIN || sf.faceId > ADFB_KMAX) return fail("adfb_block_set_bc: bad faceId %d", sf.faceId);
        if (sf.bcType < ADFB_BC_SYMM || sf.bcType > ADFB_BC_SYMMPOLAR) return fail("adfb_block_set_bc: unsupported bcType %d", sf.bcType);
        const size_t n = (size_t)(sf.icEnd - sf.icBeg + 1) * (sf.jcEnd - sf.jcBeg + 1);
        auto up = [&](const double*& hp, int ncomp) -> int {
            if (!hp) return 0;
            void* q = nullptr;
            if (cudaMalloc(&q, n * ncomp * 8) != cudaSuccess) return fail("adfb_block_set_bc: cudaMalloc failed");
            b->bcAllocs.push_back(q);
            if (cudaMemcpy(q, hp, n * ncomp * 8, cudaMemcpyHostToDevice) != cudaSuccess) return fail("adfb_block_set_bc: copy failed");
            hp = (const double*)q;  // from here on the subface holds DEVICE pointers
            return 0;
        };
        if (up(sf.norm, 3) || up(sf.rface, 1) || up(sf.uSlip, 3) || up(sf.TNSWall, 1)) return 1;
        if (up(sf.ps, 1) || up(sf.rho, 1) || up(sf.velx, 1) || up(sf.vely, 1) || up(sf.velz, 1) || up(sf.ptInlet, 1) || up(sf.ttInlet, 1) ||
            up(sf.htInlet, 1) || up(sf.flowXdirInlet, 1) || up(sf.flowYdirInlet, 1) || up(sf.flowZdirInlet, 1) || up(sf.turbInlet, 1))
            return 1;
        if (sf.bcType == ADFB_BC_SUBSONIC_OUTFLOW && !sf.ps) return fail("adfb_block_set_bc: subsonic outflow needs ps");
        if (sf.bcType == ADFB_BC_SUPERSONIC_INFLOW && !(sf.ps && sf.rho && sf.velx && sf.vely && sf.velz))
            return fail("adfb_block_set_bc: supersonic inflow needs rho, velx, vely, velz, ps");
        if (sf.bcType == ADFB_BC_SUBSONIC_INFLOW) {
            if (sf.subsonicInletTreatment == 1) {
                if (!(sf.ptInlet && sf.ttInlet && sf.htInlet && sf.flowXdirInlet && sf.flowYdirInlet && sf.flowZdirInlet))
                    return fail("adfb_block_set_bc: subsonic inflow (totalConditions) needs ptInlet, ttInlet, htInlet, flow?dirInlet");
            } else if (sf.subsonicInletTreatment == 2) {
                if (!(sf.rho && sf.velx && sf.vely && sf.velz)) return fail("adfb_block_set_bc: subsonic inflow (massFlow) needs rho, velx, vely, velz");
            } else return fail("adfb_block_set_bc: subsonicInletTreatment must be 1 (totalConditions) or 2 (massFlow)");
        }
        b->subfaces.push_back(sf);
    }
    return 0;
}

int adfb_upload_state(int blk, const double* w, const double* p) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_upload_state: no block %d", blk);
    if (!w) return fail("adfb_upload_state: w is required");
    if (put(*b, C2, b->dev.w, w, b->nw, 8)) return 1;
    if (p && put(*b, C2, b->dev.p, p, 1, 8)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

int adfb_upload_visc(int blk, const double* rlv, const double* rev) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_upload_visc: no block %d", blk);
    if (rlv && put(*b, C2, b->dev.rlv, rlv, 1, 8)) return 1;
    if (rev && put(*b, C2, b->dev.rev, rev, 1, 8)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

int adfb_download_state(int blk, double* w, double* p, double* rlv, double* rev) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_download_state: no block %d", blk);
    if (w && get(*b, C2, b->dev.w, w, b->nw, 8)) return 1;
    if (p && get(*b, C2, b->dev.p, p, 1, 8)) return 1;
    if (rlv && get(*b, C2, b->dev.rlv, rlv, 1, 8)) return 1;
    if (rev && get(*b, C2, b->dev.rev, rev, 1, 8)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

int adfb_download_residual(int blk, double* dw) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_download_residual: no block %d", blk);
    if (!dw) return fail("adfb_download_residual: null");
    if (get(*b, C2, b->dev.dw, dw, b->nw, 8)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

int adfb_download_intermed(int blk, double* dtl, double* radI, double* radJ, double* radK) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_download_intermed: no block %d", blk);
    if (dtl && get(*b, C1, b->dev.dtl, dtl, 1, 8)) return 1;
    if (radI && get(*b, C1, b->dev.radI, radI, 1, 8)) return 1;
    if (radJ && get(*b, C1, b->dev.radJ, radJ, 1, 8)) return 1;
    if (radK && get(*b, C1, b->dev.radK, radK, 1, 8)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

// debug/test access to device-resident work arrays (nodal gradients etc.)
int adfb_download_array(int blk, const char* name, double* out) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_download_array: no block %d", blk);
    const BlockDev& v = b->dev;
    const void* src = nullptr;
    int nc = 1;
    std::string s(name ? name : "");
    if (s == "grad") { src = v.grad; nc = 12; }
    else if (s == "dss") { src = v.dss; nc = 3; }
    else if (s == "ss") src = v.ss;
    else if (s == "aa") src = v.aa;
    else if (s == "si") { src = v.si; nc = 3; }
    else if (s == "sj") { src = v.sj; nc = 3; }
    else if (s == "sk") { src = v.sk; nc = 3; }
    else if (s == "fw") { src = v.fw; nc = 5; }
    else if (s == "shock") src = v.shock;
    else if (s == "dtl") src = v.dtl;
    else if (s == "radI") src = v.radI;
    else if (s == "radJ") src = v.radJ;
    else if (s == "radK") src = v.radK;
    else if (s == "wr") { src = v.wr; nc = 5; }
    else if (s == "w1") { src = v.w1; nc = 5; }
    else if (s == "p1") src = v.p1;
    else return fail("adfb_download_array: unknown array '%s'", s.c_str());
    if (get(*b, C2, src, out, nc, 8)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

long long adfb_state_size(void) {
    long long n = 0;
    for (Block& b : g.blocks)
        if (b.alive && b.level == 1) n += (long long)b.d.nx * b.d.ny * b.d.nz * b.nw;
    return n;
}

static int vec_io(double* host, long long n, int mode) {
    NEED_INIT();
    const long long need = adfb_state_size();
    if (!host || n != need) return fail("vector length %lld does not match the local state size %lld", n, need);
    if (g.dVecN < (size_t)need) {
        if (g.dVec) cudaFree(g.dVec);
        g.dVec = nullptr; g.dVecN = 0;
        CK(cudaMalloc((void**)&g.dVec, need * sizeof(double)));
        g.dVecN = need;
    }
    if (mode == 1) CK(cudaMemcpyAsync(g.dVec, host, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    long long off = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        if (launch_vec(b.d, b.dev, b.nw, g.dVec + off, mode, g.stream)) return fail("vector kernel launch failed");
        off += (long long)b.d.nx * b.d.ny * b.d.nz * b.nw;
    }
    if (mode != 1) CK(cudaMemcpyAsync(host, g.dVec, need * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int adfb_get_states(double* states, long long n) { return vec_io(states, n, 0); }
int adfb_set_states(const double* states, long long n) { return vec_io((double*)states, n, 1); }
int adfb_get_res(double* res, long long n) { return vec_io(res, n, 2); }

// ---------------------------------------------------------------------------
// halo exchange
}  // extern "C" (templates need C++ linkage)
static Context::Pattern* g_upPat = nullptr;   // pattern that owns the uploads of the current set call
template <typename T>
static int pat_upload(T** dst, const std::vector<T>& src) {
    *dst = nullptr;
    if (src.empty()) return 0;
    void* q = nullptr;
    if (cudaMalloc(&q, src.size() * sizeof(T)) != cudaSuccess) return fail("comm pattern: cudaMalloc failed");
    if (!g_upPat) { cudaFree(q); return fail("comm pattern: internal error (no upload target)"); }
    g_upPat->allocs.push_back(q);
    if (cudaMemcpy(q, src.data(), src.size() * sizeof(T), cudaMemcpyHostToDevice) != cudaSuccess) return fail("comm pattern: copy failed");
    *dst = (T*)q;
    return 0;
}

static int list_to_offsets(const int* list, long long n, std::vector<int>& blk, std::vector<long long>& off, const char* what) {
    blk.resize(n); off.resize(n);
    for (long long e = 0; e < n; e++) {
        const int bId = list[4 * e], i = list[4 * e + 1], j = list[4 * e + 2], k = list[4 * e + 3];
        Block* b = get_block(bId);
        if (!b) return fail("adfb_comm_set_pattern: %s entry %lld names unknown block %d", what, e, bId);
        const Dims& d = b->d;
        if (i < 0 || i > d.ib || j < 0 || j > d.jb || k < 0 || k > d.kb)
            return fail("adfb_comm_set_pattern: %s entry %lld index (%d,%d,%d) outside block %d", what, e, i, j, k, bId);
        blk[e] = bId;
        off[e] = ADFB_IDX(i, j, k);
    }
    return 0;
}

static int set_pattern_impl(Context::Pattern& P, int nNbr, const int* nbrRank, const int* sendCount, const int* recvCount,
                            const int* sendList, const double* sendInterp, const int* recvList, int nInternal,
                            const int* donorList, const double* donorInterp, const int* haloList, bool interp) {
    if (nNbr < 0 || nInternal < 0) return fail("adfb_comm_set_pattern: negative counts");
    drop_graphs();
    if (nNbr > 0 && g.nranks == 1) return fail("adfb_comm_set_pattern: neighbour ranks given but adfb_init was called with nranks = 1");
    if (cudaStreamSynchronize(g.stream) != cudaSuccess) return fail("stream sync failed");
    for (void* q : P.allocs) cudaFree(q);
    P = Context::Pattern();
    P.interp = interp;
    g_upPat = &P;
    std::vector<long long> cumS, cumR;
    std::vector<int> locS, locR, cntS, cntR;
    for (int m = 0; m < nNbr; m++) {
        if (nbrRank[m] < 0 || nbrRank[m] >= g.nranks || nbrRank[m] == g.rank) return fail("adfb_comm_set_pattern: bad neighbour rank %d", nbrRank[m]);
        P.nbrRank.push_back(nbrRank[m]); P.sendCount.push_back(sendCount[m]); P.recvCount.push_back(recvCount[m]);
        for (int e = 0; e < sendCount[m]; e++) { cumS.push_back(P.nSend); locS.push_back(e); cntS.push_back(sendCount[m]); }
        for (int e = 0; e < recvCount[m]; e++) { cumR.push_back(P.nRecv); locR.push_back(e); cntR.push_back(recvCount[m]); }
        P.nSend += sendCount[m]; P.nRecv += recvCount[m];
    }
    P.nInt = nInternal;
    std::vector<int> blk; std::vector<long long> off;
    // donor entries of an overset pattern: all 8 cells (i..i+1, ...) must exist, and the block strides travel along
    auto donor_extra = [&](const int* list, long long n, const double* w, long long** dSJ, long long** dSK, double** dW, const char* what) -> int {
        if (!w) return fail("adfb_comm_set_overset: %s interpolation weights missing", what);
        std::vector<long long> sj(n), sk(n);
        for (long long e = 0; e < n; e++) {
            Block* b = get_block(list[4 * e]);
            const Dims& d = b->d;
            if (list[4 * e + 1] + 1 > d.ib || list[4 * e + 2] + 1 > d.jb || list[4 * e + 3] + 1 > d.kb)
                return fail("adfb_comm_set_overset: %s entry %lld: donor stencil leaves block %d", what, e, list[4 * e]);
            sj[e] = d.sJ; sk[e] = d.sK;
        }
        std::vector<double> wv(w, w + 8 * n);
        return pat_upload(dSJ, sj) || pat_upload(dSK, sk) || pat_upload(dW, wv);
    };
    if (P.nSend) {
        if (list_to_offsets(sendList, P.nSend, blk, off, "send")) return 1;
        if (pat_upload(&P.sBlk, blk) || pat_upload(&P.sOff, off) || pat_upload(&P.sCum, cumS) || pat_upload(&P.sLocal, locS) || pat_upload(&P.sCount, cntS)) return 1;
        if (interp && donor_extra(sendList, P.nSend, sendInterp, &P.sSJ, &P.sSK, &P.sW, "send")) return 1;
    }
    if (P.nRecv) {
        if (list_to_offsets(recvList, P.nRecv, blk, off, "recv")) return 1;
        if (pat_upload(&P.rBlk, blk) || pat_upload(&P.rOff, off) || pat_upload(&P.rCum, cumR) || pat_upload(&P.rLocal, locR) || pat_upload(&P.rCount, cntR)) return 1;
    }
    if (P.nInt) {
        if (list_to_offsets(donorList, P.nInt, blk, off, "donor")) return 1;
        if (pat_upload(&P.iSrcBlk, blk) || pat_upload(&P.iSrcOff, off)) return 1;
        if (interp && donor_extra(donorList, P.nInt, donorInterp, &P.iSJ, &P.iSK, &P.iW, "donor")) return 1;
        if (list_to_offsets(haloList, P.nInt, blk, off, "halo")) return 1;
        if (pat_upload(&P.iDstBlk, blk) || pat_upload(&P.iDstOff, off)) return 1;
    }
    void* q = nullptr;
    if (P.nSend) { if (cudaMalloc(&q, (size_t)P.nSend * ADFB_MAX_COMM_VARS * 8) != cudaSuccess) return fail("comm pattern: cudaMalloc failed"); P.allocs.push_back(q); P.sendBuf = (double*)q; }
    if (P.nRecv) { if (cudaMalloc(&q, (size_t)P.nRecv * ADFB_MAX_COMM_VARS * 8) != cudaSuccess) return fail("comm pattern: cudaMalloc failed"); P.allocs.push_back(q); P.recvBuf = (double*)q; }
    P.tabBlocks = (int)g.blocks.size();
    P.set = true;
    g_upPat = nullptr;
    return 0;
}

extern "C" {
int adfb_comm_set_pattern(int level, int nNbr, const int* nbrRank, const int* sendCount, const int* recvCount,
                          const int* sendList, const int* recvList, int nInternal, const int* donorList,
                          const int* haloList) {
    NEED_INIT();
    return set_pattern_impl(g.pats[level], nNbr, nbrRank, sendCount, recvCount, sendList, nullptr, recvList, nInternal, donorList, nullptr,
                            haloList, false);
}
int adfb_comm_set_overset(int level, int nNbr, const int* nbrRank, const int* sendCount, const int* recvCount,
                          const int* sendList, const double* sendInterp, const int* recvList, int nInternal,
                          const int* donorList, const double* donorInterp, const int* haloList) {
    NEED_INIT();
    return set_pattern_impl(g.ovPats[level], nNbr, nbrRank, sendCount, recvCount, sendList, sendInterp, recvList, nInternal, donorList,
                            donorInterp, haloList, true);
}

// whalo1to1 part of whalo2/whalo1 for the variable selection of setCommPointers
// (src/utils/haloExchange.F90:356-470)
extern "C" int adfb_block_set_orphans(int blk, int nOrphans, const int32_t* orphans, double muInf, double eddyVisInfRatio) {
    NEED_INIT();
    Block* b = get_block(blk);
    if (!b) return fail("adfb_block_set_orphans: no block %d", blk);
    if (nOrphans < 0 || (nOrphans > 0 && !orphans)) return fail("adfb_block_set_orphans: bad arguments");
    drop_graphs();
    cudaStreamSynchronize(g.stream);
    if (b->dOrphans) { cudaFree(b->dOrphans); b->dOrphans = nullptr; }
    b->nOrphans = 0;
    for (int n = 0; n < nOrphans; n++) {
        const int i = orphans[3 * n], j = orphans[3 * n + 1], k = orphans[3 * n + 2];
        if (i < 0 || i > b->d.ib || j < 0 || j > b->d.jb || k < 0 || k > b->d.kb)
            return fail("adfb_block_set_orphans: orphan %d (%d, %d, %d) outside the block", n, i, j, k);
    }
    if (nOrphans > 0) {
        CK(cudaMalloc((void**)&b->dOrphans, (size_t)3 * nOrphans * sizeof(int32_t)));
        CK(cudaMemcpy(b->dOrphans, orphans, (size_t)3 * nOrphans * sizeof(int32_t), cudaMemcpyHostToDevice));
    }
    b->nOrphans = nOrphans; b->muInf = muInf; b->eddyVisInfRatio = eddyVisInfRatio;
    return 0;
}

// phase 0: the whole exchange on the compute stream.  Phases 1 / 2 split it so that the transfer overlaps the boundary
// conditions (the reference posts its receives and sends, then copies locally, then waits: haloExchange.F90:620-716):
//   1 "post"   : pack the send lists of the 1-to-1 pattern (owned cells only: the BCs that follow do not touch them) and
//                run the grouped ncclSend/ncclRecv on the communication stream
//   2 "finish" : join the communication stream, same-rank copies, unpack, then the overset pattern and the owned-cell
//                total energy -- after the BCs, like the un-split order (edge halos of the BCs read the OLD interface halos)
static bool halo_split_ok(int level) {
    static int on = -1;
    if (on < 0) { const char* e = getenv("ADFB_HALO_OVERLAP"); on = e ? atoi(e) : 1; }
    if (!on || g_kt.on || g.nranks < 2) return false;
    auto it = g.pats.find(level);
    return it != g.pats.end() && it->second.set && !it->second.nbrRank.empty();
}
static int halo_exchange_impl(int level, int start, int end, int commPressure, int commViscous, bool etotOwned, int phase = 0) {
    const bool viscous = g.prm.equations != ADFB_EULER, eddy = g.prm.equations == ADFB_RANS;
    // whalo1to1 with commPatternCell_2nd / internalCell_2nd, then wOverset with commPatternOverset / internalOverset
    // (whalo2, haloExchange.F90:139-146); orphan averaging is not supported (nOrphans must be 0)
    Context::Pattern* both[2] = {nullptr, nullptr};
    { auto it = g.pats.find(level); if (it != g.pats.end()) both[0] = &it->second; }
    { auto it = g.ovPats.find(level); if (it != g.ovPats.end()) both[1] = &it->second; }
    for (Context::Pattern* PP : both) {
        if (!PP) continue;
        Context::Pattern& P = *PP;
        if (!(P.set && (P.nSend || P.nRecv || P.nInt))) continue;
        const bool oneToOne = PP == both[0];
        if (phase == 1 && !oneToOne) continue;           // the overset pattern is exchanged in one piece by "finish"
        const bool doPost = phase == 0 || phase == 1 || !oneToOne;      // pack + send/recv
        const bool doFinish = phase == 0 || phase == 2;                  // local copies + unpack
        cudaStream_t cs = (phase == 1) ? g.commStream : g.stream;        // stream of pack + NCCL
        if (phase == 1) {
            CK(cudaEventRecord(g.evPost, g.stream));
            CK(cudaStreamWaitEvent(g.commStream, g.evPost, 0));
        }
        if ((int)g.blocks.size() != P.tabBlocks) return fail("halo exchange: blocks changed after adfb_comm_set_pattern");
        const int key = start | (end << 4) | ((commPressure ? 1 : 0) << 8) | ((commViscous ? 1 : 0) << 9);
        int nVar = 0;
        {
            Block* b0 = nullptr;
            for (Block& b : g.blocks) if (b.alive && b.level == level) { b0 = &b; break; }
            if (!b0) return 0;
            for (int l = start; l <= end && l <= b0->nw; l++) nVar++;
            if (commPressure) nVar++;
            if (viscous && commViscous) nVar++;
            if (eddy && commViscous) nVar++;
        }
        if (nVar == 0) return 0;
        if (nVar > ADFB_MAX_COMM_VARS) return fail("halo exchange: too many variables");
        CommVarTable* dTab = nullptr;
        auto it = P.tabs.find(key);
        if (it != P.tabs.end()) dTab = it->second;
        else {
            std::vector<CommVarTable> tab(P.tabBlocks);
            for (int bId = 0; bId < P.tabBlocks; bId++) {
                Block& b = g.blocks[bId];
                memset(&tab[bId], 0, sizeof(CommVarTable));
                if (!b.alive) continue;
                int v = 0;
                for (int l = start; l <= end && l <= b.nw; l++) tab[bId].ptr[v++] = b.dev.w + (size_t)(l - 1) * b.d.N;
                if (commPressure) tab[bId].ptr[v++] = b.dev.p;
                if (viscous && commViscous) tab[bId].ptr[v++] = b.dev.rlv;
                if (eddy && commViscous) tab[bId].ptr[v++] = b.dev.rev;
            }
            void* q = nullptr;
            CK(cudaMalloc(&q, sizeof(CommVarTable) * P.tabBlocks));
            P.allocs.push_back(q);
            CK(cudaMemcpy(q, tab.data(), sizeof(CommVarTable) * P.tabBlocks, cudaMemcpyHostToDevice));
            dTab = (CommVarTable*)q;
            P.tabs[key] = dTab;
        }
        if (doPost && P.nSend) {
            const long long n = P.nSend * nVar;
            KT_BEGIN(K_HALO, cs);
            if (P.interp)
                k_halo_pack_interp<<<(unsigned)((n + 255) / 256), 256, 0, cs>>>(P.sBlk, P.sOff, P.sCum, P.sLocal, P.sCount, P.sSJ, P.sSK,
                                                                               P.sW, dTab, nVar, P.nSend, P.sendBuf);
            else
                k_halo_pack<<<(unsigned)((n + 255) / 256), 256, 0, cs>>>(P.sBlk, P.sOff, P.sCum, P.sLocal, P.sCount, dTab, nVar, P.nSend, P.sendBuf);
            KT_END(K_HALO, cs);
        }
        if (doPost && !P.nbrRank.empty()) {
            int rc = g.nccl.GroupStart();
            long long so = 0, ro = 0;
            for (size_t m = 0; m < P.nbrRank.size() && rc == 0; m++) {
                if (P.sendCount[m]) rc = g.nccl.Send(P.sendBuf + so * nVar, (size_t)P.sendCount[m] * nVar, kNcclDouble, P.nbrRank[m], g.comm, cs);
                if (rc == 0 && P.recvCount[m]) rc = g.nccl.Recv(P.recvBuf + ro * nVar, (size_t)P.recvCount[m] * nVar, kNcclDouble, P.nbrRank[m], g.comm, cs);
                so += P.sendCount[m]; ro += P.recvCount[m];
            }
            const int rc2 = g.nccl.GroupEnd();
            if (rc != 0 || rc2 != 0) return fail("NCCL halo exchange: %s", g.nccl.GetErrorString(rc ? rc : rc2));
        }
        if (phase == 1) { CK(cudaEventRecord(g.evDone, g.commStream)); continue; }
        if (phase == 2 && oneToOne) CK(cudaStreamWaitEvent(g.stream, g.evDone, 0));
        if (!doFinish) continue;
        if (P.nInt) {
            const long long n = P.nInt * nVar;
            KT_BEGIN(K_HALO, g.stream);
            if (P.interp)
                k_halo_internal_interp<<<(unsigned)((n + 255) / 256), 256, 0, g.stream>>>(P.iSrcBlk, P.iSrcOff, P.iSJ, P.iSK, P.iW, P.iDstBlk,
                                                                                         P.iDstOff, dTab, nVar, P.nInt);
            else
                k_halo_internal<<<(unsigned)((n + 255) / 256), 256, 0, g.stream>>>(P.iSrcBlk, P.iSrcOff, P.iDstBlk, P.iDstOff, dTab, nVar, P.nInt);
            KT_END(K_HALO, g.stream);
        }
        if (P.nRecv) {
            const long long n = P.nRecv * nVar;
            KT_BEGIN(K_HALO, g.stream);
            k_halo_unpack<<<(unsigned)((n + 255) / 256), 256, 0, g.stream>>>(P.rBlk, P.rOff, P.rCum, P.rLocal, P.rCount, dTab, nVar, P.nRecv, P.recvBuf);
            KT_END(K_HALO, g.stream);
        }
    }
    // orphanAverage on every block that carries an orphan list (haloExchange.F90:56-66, :161-171)
    if (phase != 1) {
        for (Block& b : g.blocks) {
            if (!b.alive || b.level != level || b.nOrphans == 0) continue;
            const int lEnd = end < b.nw ? end : b.nw;
            KT_BEGIN(K_HALO, g.stream);
            k_orphan_average<<<(b.nOrphans + 127) / 128, 128, 0, g.stream>>>(b.d, b.dev, b.nOrphans, b.dOrphans, start, lEnd, commPressure ? 1 : 0,
                                                                             (viscous && commViscous) ? 1 : 0, (eddy && commViscous) ? 1 : 0,
                                                                             b.muInf, b.eddyVisInfRatio);
            KT_END(K_HALO, g.stream);
        }
    }
    // bothPAndE: computeEtotBlock(2, il, 2, jl, 2, kl) on every block (haloExchange.F90:174-197)
    if (phase != 1 && etotOwned && commPressure && start <= 5 && end >= 5) {
        for (Block& b : g.blocks) {
            if (!b.alive || b.level != level) continue;
            dim3 tb(32, 4, 2);
            dim3 gr((b.d.nx + 31) / 32, (b.d.ny + 3) / 4, (b.d.nz + 1) / 2);
            KT_BEGIN(K_HALO, g.stream);
            k_etot_owned<<<gr, tb, 0, g.stream>>>(b.d, b.dev);
            KT_END(K_HALO, g.stream);
        }
    }
    CK(cudaGetLastError());
    return 0;
}

int adfb_halo_exchange(int level, int start, int end, int commPressure, int commGamma, int commViscous) {
    ADFB_RANGE("adfb_halo_exchange");
    NEED_INIT();
    (void)commGamma;  // gamma is constant (cpConstant): commVarGamma is always false, haloExchange.F90:146
    if (!g.havePrm) return fail("adfb_halo_exchange: adfb_set_params has not been called");
    if (start < 1 || end > 6 || (end >= start && false)) return fail("adfb_halo_exchange: bad variable range %d:%d", start, end);
    return halo_exchange_impl(level, start, end, commPressure, commViscous, true);
}

static int residual_body(int level, unsigned flags);
// an overset pattern with entries exists on this level: whalo2 then really changes rhoE of fringe cells
// (computeEtotBlock after wOverset, haloExchange.F90:174-197), so the owned-cell etot pass is not idempotent
static bool overset_present(int level) {
    auto it = g.ovPats.find(level);
    return it != g.ovPats.end() && it->second.set && (it->second.nSend || it->second.nRecv || it->second.nInt);
}
int adfb_residual(int level, unsigned flags) {
    ADFB_RANGE("adfb_residual");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_residual: adfb_set_params has not been called");
    if (!(flags & (ADFB_RES_FLOW | ADFB_RES_TURB))) return fail("adfb_residual: neither flow nor turbulence residual requested");
    for (Block& b : g.blocks)
        if (b.alive && b.level == level && !b.haveMetrics) return fail("adfb_residual: geometry of a block was never set");
    const unsigned long long key = (1ull << 40) | ((unsigned long long)level << 32) | flags | (g.mffdFuse ? (1ull << 31) : 0ull);
    return run_graphed(key, [&]() { return residual_body(level, flags); });
}

static int residual_body(int level, unsigned flags) {
    if (!(flags & ADFB_RES_SKIP_PREAMBLE)) {
        for (Block& b : g.blocks) {
            if (!b.alive || b.level != level) continue;
            // blocketteRes :213-226: p, rlv, rev on owned cells, then turbulence and flow BCs
            if (!g.mffdFuse && launch_state_prep(b.d, b.dev, g.prm, false, (flags & ADFB_RES_FLOW) != 0, g.stream)) return fail("state prep launch failed");
        }
        // whalo2(1, lStart, lEnd, T, T, T), blockette.F90:231-246; the owned-cell
        // computeEtotBlock of whalo2 is fused into k_state_prep (see DESIGN.md).  Multi-rank: the send lists (owned cells)
        // are packed and sent while the BC chain runs; the halos are written after it.
        const int nwLoc = g.prm.equations == ADFB_RANS ? 6 : 5;
        const bool fr = flags & ADFB_RES_FLOW, tr = (flags & ADFB_RES_TURB) && nwLoc == 6;
        const int lStart = fr ? 1 : 6, lEnd = tr ? 6 : 5;
        const bool ov = overset_present(level);
        const bool split = halo_split_ok(level);
        if (split && halo_exchange_impl(level, lStart, lEnd, 1, 1, ov, 1)) return 1;
        for (Block& b : g.blocks) {
            if (!b.alive || b.level != level) continue;
            if (launch_bc_levels(b.d, b.dev, b.subfaces, 1, g.prm.equations == ADFB_RANS && (flags & ADFB_RES_TURB), 1, g.stream))
                return fail("BC launch failed");
        }
        if (halo_exchange_impl(level, lStart, lEnd, 1, 1, ov, split ? 2 : 0)) return 1;
        if (ov) {
            // blocketteRes re-applies the turbulence and flow BCs on every block after whalo2 when overset blocks are
            // present (blockette.F90:252-262): boundary halos next to fringe cells see the interpolated values
            for (Block& b : g.blocks) {
                if (!b.alive || b.level != level) continue;
                if (launch_bc_levels(b.d, b.dev, b.subfaces, 1, g.prm.equations == ADFB_RANS && (flags & ADFB_RES_TURB), 1, g.stream))
                    return fail("BC launch failed");
            }
        }
    }
    long long cell0 = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        const MffdEpi mf = {g.mffdFuse ? g.dMffd : nullptr, cell0};
        if (launch_residual_core(b.d, b.dev, g.prm, g.env, residual_discr(level, true), flags, 1.0, 0, 1, g.stream, 0, mf))
            return fail("residual kernel launch failed: %s", cudaGetErrorString(cudaGetLastError()));
        cell0 += (long long)b.d.nx * b.d.ny * b.d.nz;
    }
    CK(cudaGetLastError());
    return 0;
}

// ---------------------------------------------------------------------------
// NK matrix-free residual-Jacobian product (src/NKSolver/NKSolvers.F90:437-461, :1331-1376,
// :1262-1329; PETSc MatMFFD y = (F(U + h a) - F(U)) / h)
static int nk_buffers(long long need) {
    if (g.nkN >= (size_t)need) return 0;
    for (double** p : {&g.nkA, &g.nkU, &g.nkF0, &g.nkY}) { if (*p) cudaFree(*p); *p = nullptr; }
    g.nkN = 0;
    g.nkHaveBase = false; g.ankHaveBase = false; g.ankTurbHaveBase = false;   // the base vectors went with the buffers
    for (double** p : {&g.nkA, &g.nkU, &g.nkF0, &g.nkY}) CK(cudaMalloc((void**)p, need * sizeof(double)));
    if (!g.dRed) { CK(cudaMalloc((void**)&g.dRed, (2 * 1024 + 2) * sizeof(double))); g.dRedN = 2 * 1024 + 2; }
    g.nkN = need;
    return 0;
}
static int nk_vec_kernel(const double* vec, const double* base, double* out, double h, int mode) {
    long long off = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        const long long n = (long long)b.d.nx * b.d.ny * b.d.nz * b.nw;
        KT_BEGIN(K_MFFD, g.stream);
        k_nkvec<<<(unsigned)((n + 255) / 256), 256, 0, g.stream>>>(b.d, b.dev, b.nw, vec ? vec + off : nullptr, base ? base + off : nullptr,
                                                                   out ? out + off : nullptr, h, mode, 0LL, LLONG_MAX);
        KT_END(K_MFFD, g.stream);
        off += n;
    }
    CK(cudaGetLastError());
    return 0;
}
// sum of squares of a device vector, all-reduced; result in *out
static int nk_sumsq(const double* v, long long n, double* out) {
    const int nPart = 512;
    KT_BEGIN(K_MFFD, g.stream);
    k_sumsq_partial<<<nPart, 256, 0, g.stream>>>(v, n, g.dRed);
    KT_END(K_MFFD, g.stream);
    KT_BEGIN(K_MFFD, g.stream);
    k_sum_final<<<1, 256, 0, g.stream>>>(g.dRed, nPart);
    KT_END(K_MFFD, g.stream);
    if (g.nranks > 1) {
        const int rc = g.nccl.AllReduce(g.dRed + nPart, g.dRed + nPart, 1, kNcclDouble, kNcclSum, g.comm, g.stream);
        if (rc != 0) return fail("ncclAllReduce: %s", g.nccl.GetErrorString(rc));
    }
    CK(cudaMemcpyAsync(g.hRed, g.dRed + nPart, sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    *out = g.hRed[0];
    return 0;
}
static const unsigned kNkFlags = ADFB_RES_FLOW | ADFB_RES_TURB;

// FormFunction_mf as a slab pipeline.  The state vector is ordered with k slowest, so a range of k planes is a contiguous piece of
// wVec / rVec.  Every stage of blocketteRes is local in k up to +-2 planes -- setW and the p / rlv / rev preamble are cell local,
// an i- or j-face boundary cell touches its own plane only (launch_bc_levels), the time-step / sensor preparation is cell
// local, the SA row and the tile kernel read two planes either side -- so the residual of the planes of slab s can be formed
// as soon as slab s+1 has arrived, while later slabs are still on the bus, and its rows leave while the next ones are computed:
// the host-to-device copy, the kernels and the device-to-host copy of one call overlap (three streams, full-duplex PCIe).
// Same kernels, same operands as the one-shot path: the result is identical.  Used when both vectors are page-locked, the
// blocks have no exchange partners (no 1-to-1 / overset pattern on level 1) and the tile kernel applies; ADFB_FF_PIPE=0 disables it.
static bool ff_pinned(const void* p) {
    cudaPointerAttributes a;
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return false; }
    return a.type == cudaMemoryTypeHost;
}
static int form_function_pipe_slabs() {   // read at every call: tests switch it
    const char* e = getenv("ADFB_FF_PIPE");
    return e ? atoi(e) : 6;   // C2 on one H100 SXM (400 W limit): 4 / 6 / 8 / 12 slabs 0.87 / 0.75 / 0.78 / 0.74 ms per call
}
// the stream work of one pipelined call (captured into a CUDA graph per (wVec, rVec) pair: ~15 launches per slab otherwise
// cost more host time than the GPU needs for them).  Front end of a slab (setW, p / rlv / rev, BCs, time step / sensor) on the
// library stream, back end (SA row, tile kernel, setRVec) on a second one: the front end of slab s+1 touches planes above the
// ones the back end of slab s reads, so the two run side by side.
static const int kFfPlanesPerCta = 4;   // k planes per CTA of the tile kernel inside the pipeline
static int form_function_pipe_body(const double* wVec, double* rVec, int wantSlabs) {
    const int kc = kFfPlanesPerCta;
    const bool rans = g.prm.equations == ADFB_RANS;
    cudaStream_t sF = g.stream, sB = g.ffBack;
    // fork: the other streams start after whatever the library stream still has in flight
    CK(cudaEventRecord(g.ffEv[3][0], sF));
    CK(cudaStreamWaitEvent(g.ffIn, g.ffEv[3][0], 0));
    CK(cudaStreamWaitEvent(g.ffOut, g.ffEv[3][0], 0));
    CK(cudaStreamWaitEvent(sB, g.ffEv[3][0], 0));
    long long off = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        const Dims& d = b.d;
        const long long plane = (long long)d.nx * d.ny * b.nw;   // vector entries per k plane
        const int nChunks = (d.nz + kc - 1) / kc;
        const int S = std::min(std::min(wantSlabs, 32), nChunks / 2);
        // slab boundaries in chunks: small slabs at both ends (the pipeline fills and drains faster), larger ones in the middle
        std::vector<int> cb(S + 1, 0);
        {
            std::vector<double> wgt(S);
            double tot = 0.0;
            for (int q = 0; q < S; q++) { const double x = (q + 0.5) / S; wgt[q] = 0.6 + 3.2 * x * (1.0 - x); tot += wgt[q]; }
            double acc = 0.0;
            for (int q = 0; q < S; q++) {
                acc += wgt[q];
                int e = (int)(acc / tot * nChunks + 0.5);
                if (e <= cb[q]) e = cb[q] + 1;
                if (e > nChunks - (S - 1 - q)) e = nChunks - (S - 1 - q);
                cb[q + 1] = e;
            }
            cb[S] = nChunks;
        }
        auto ownedEnd = [&](int chunkEnd) { return std::min(chunkEnd * kc, d.nz); };   // owned plane index (0-based), exclusive
        for (int q = 0; q < S; q++) {   // all host-to-device copies are queued at once; they run back to back on their stream
            const long long q0 = (long long)ownedEnd(cb[q]) * plane, q1 = (long long)ownedEnd(cb[q + 1]) * plane;
            CK(cudaMemcpyAsync(g.nkA + off + q0, wVec + off + q0, (size_t)(q1 - q0) * sizeof(double), cudaMemcpyHostToDevice, g.ffIn));
            CK(cudaEventRecord(g.ffEv[0][q], g.ffIn));
        }
        int cNext = 0;   // first k chunk whose residual has not been formed
        for (int q = 0; q < S; q++) {
            const bool first = q == 0, last = q == S - 1;
            const int o0 = ownedEnd(cb[q]), o1 = ownedEnd(cb[q + 1]);   // owned planes o0 .. o1-1 (0-based) = absolute 2+o0 .. 1+o1
            CK(cudaStreamWaitEvent(sF, g.ffEv[0][q], 0));
            // setW + p / rlv / rev of the slab's owned cells
            {
                const long long q0 = (long long)o0 * plane, q1 = (long long)o1 * plane;
                KT_BEGIN(K_MFFD, sF);
                k_nkvec<<<(unsigned)((q1 - q0 + 255) / 256), 256, 0, sF>>>(d, b.dev, b.nw, g.nkA + off, nullptr, nullptr, 0.0, 0, q0, q1);
                KT_END(K_MFFD, sF);
                dim3 tb(32, 4, 2);
                dim3 gr((d.nx + 31) / 32, (d.ny + 3) / 4, (o1 - o0 + 1) / 2);
                KT_BEGIN(K_STATE, sF);
                launch_pdl(k_state_prep, gr, tb, sF, d, b.dev, 0, rans ? 6 : 5, 1, o0, 1 + o1);
                KT_END(K_STATE, sF);
            }
            // boundary conditions of the slab's planes (+ the k-face subfaces with the first / last slab)
            const int pLo = first ? 0 : 2 + o0, pHi = last ? d.kb : 1 + o1;
            if (launch_bc_levels(d, b.dev, b.subfaces, 1, rans ? 1 : 0, 1, sF, first ? -(1 << 30) : pLo, last ? (1 << 30) : pHi,
                                 (first ? 1 : 0) | (last ? 2 : 0)))
                return fail("BC launch failed");
            // time step / radii / sensor of the slab's planes (halo planes with the first and the last slab)
            {
                dim3 tb(32, 4, 2);
                dim3 gr((d.NI + 31) / 32, (d.NJ + 3) / 4, (pHi - pLo + 2) / 2);
                KT_BEGIN(K_PREP, sF);
                launch_pdl(k_prep, gr, tb, sF, d, b.dev, 1, 1, pLo, pHi, residual_discr(1, true), 1);
                KT_END(K_PREP, sF);
            }
            // residual rows of the k chunks whose +-2 plane stencil is complete
            int cEnd = cNext;
            while (cEnd < nChunks && (last || 2 + ownedEnd(cEnd + 1) - 1 + 2 <= pHi)) cEnd++;
            if (cEnd > cNext) {
                CK(cudaEventRecord(g.ffEv[2][q], sF));
                CK(cudaStreamWaitEvent(sB, g.ffEv[2][q], 0));
                const int r0 = ownedEnd(cNext), r1 = ownedEnd(cEnd);
                if (rans) {
                    dim3 tr(32, 4, 1);
                    dim3 gr((d.nx + 31) / 32, (d.ny + 3) / 4, r1 - r0);
                    KT_BEGIN(K_SA, sB);
                    k_sa<<<gr, tr, 0, sB>>>(d, b.dev, MffdEpi{nullptr, 0}, r0, 1 + r1);
                    KT_END(K_SA, sB);
                }
                KT_BEGIN(K_RESID, sB);
                const int rc = launch_flowres_tile(d, b.dev, g.prm, g.env, (int)((b.dev.p - b.dev.w) / d.N), 1.0, 1, true, 0, sB, MffdEpi{nullptr, 0},
                                                   kc, cNext, cEnd - cNext);
                KT_END(K_RESID, sB);
                if (rc) return fail("tile kernel launch failed inside the form-function pipeline");
                const long long q0 = (long long)r0 * plane, q1 = (long long)r1 * plane;
                KT_BEGIN(K_MFFD, sB);
                k_nkvec<<<(unsigned)((q1 - q0 + 255) / 256), 256, 0, sB>>>(d, b.dev, b.nw, nullptr, nullptr, g.nkY + off, 1.0, 2, q0, q1);
                KT_END(K_MFFD, sB);
                CK(cudaEventRecord(g.ffEv[1][q], sB));
                CK(cudaStreamWaitEvent(g.ffOut, g.ffEv[1][q], 0));
                CK(cudaMemcpyAsync(rVec + off + q0, g.nkY + off + q0, (size_t)(q1 - q0) * sizeof(double), cudaMemcpyDeviceToHost, g.ffOut));
                cNext = cEnd;
            }
        }
        off += (long long)d.nz * plane;
    }
    // join: everything meets on the library stream again
    CK(cudaEventRecord(g.ffEv[3][1], g.ffIn));
    CK(cudaStreamWaitEvent(sF, g.ffEv[3][1], 0));
    CK(cudaEventRecord(g.ffEv[3][2], g.ffOut));
    CK(cudaStreamWaitEvent(sF, g.ffEv[3][2], 0));
    CK(cudaEventRecord(g.ffEv[3][3], sB));
    CK(cudaStreamWaitEvent(sF, g.ffEv[3][3], 0));
    CK(cudaGetLastError());
    return 0;
}
// returns -1 when the pipeline does not apply (caller takes the one-shot path)
static int form_function_pipelined(const double* wVec, double* rVec, long long need) {
    (void)need;
    const int wantSlabs = form_function_pipe_slabs();
    if (wantSlabs < 2 || g.nranks > 1 || g_kt.on || g.mffdFuse) return -1;
    {   // exchange partners (entries in a 1-to-1 or overset pattern of level 1) tie planes of different slabs together
        auto busy = [](const std::map<int, Context::Pattern>& m) {
            auto it = m.find(1);
            return it != m.end() && it->second.set && (it->second.nSend || it->second.nRecv || it->second.nInt);
        };
        if (busy(g.pats) || busy(g.ovPats)) return -1;
    }
    if (!ff_pinned(wVec) || !ff_pinned(rVec)) return -1;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        if (!b.haveMetrics || b.nOrphans || !tile_kernel_applies(b.d, b.dev, residual_discr(1, true)) || b.d.nz < 16) return -1;
    }
    // one graph per (wVec, rVec, slabs): an NK solve calls with the same PETSc vectors over and over
    unsigned long long h = 1469598103934665603ull;
    for (unsigned long long v : {(unsigned long long)(uintptr_t)wVec, (unsigned long long)(uintptr_t)rVec, (unsigned long long)wantSlabs})
        h = (h ^ v) * 1099511628211ull;
    const unsigned long long key = (12ull << 40) | (h & 0xffffffffffull);
    {   // a handful of vector pairs at most: forget the oldest graph beyond that
        std::vector<unsigned long long>& keys = g.ffKeys;
        if (std::find(keys.begin(), keys.end(), key) == keys.end()) {
            keys.push_back(key);
            if (keys.size() > 8) {
                auto it = g.graphs.find(keys.front());
                if (it != g.graphs.end()) { cudaGraphExecDestroy(it->second); g.graphLaunches.erase(it->first); g.graphs.erase(it); }
                keys.erase(keys.begin());
            }
        }
    }
    const int rc = run_graphed(key, [&]() { return form_function_pipe_body(wVec, rVec, wantSlabs); });
    if (rc) return rc;
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

// FormFunction_mf (NKSolvers.F90:437-461): setW(wVec); computeResidualNK; setRVec(rVec)
int adfb_form_function(const double* wVec, double* rVec, long long n) {
    ADFB_RANGE("adfb_form_function");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_form_function: adfb_set_params has not been called");
    const long long need = adfb_state_size();
    if (!wVec || !rVec || n != need) return fail("adfb_form_function: vector length %lld != local state size %lld", n, need);
    if (nk_buffers(need)) return 1;
    for (Block& b : g.blocks)
        if (b.alive && b.level == 1 && !b.haveMetrics) return fail("adfb_form_function: geometry of a block was never set");
    {
        const int rc = form_function_pipelined(wVec, rVec, need);
        if (rc >= 0) return rc;
    }
    CK(cudaMemcpyAsync(g.nkA, wVec, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (nk_vec_kernel(g.nkA, nullptr, nullptr, 0.0, 0)) return 1;
    if (adfb_residual(1, kNkFlags)) return 1;
    if (nk_vec_kernel(nullptr, nullptr, g.nkY, 1.0, 2)) return 1;
    CK(cudaMemcpyAsync(rVec, g.nkY, need * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}

// MatMFFDSetBase(dRdw, wVec, baseRes) (NKSolvers.F90:628-630): U <- wVec, F0 <- F(U) on the device
int adfb_mffd_set_base(const double* U, long long n) {
    ADFB_RANGE("adfb_mffd_set_base");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_mffd_set_base: adfb_set_params has not been called");
    const long long need = adfb_state_size();
    if (!U || n != need) return fail("adfb_mffd_set_base: vector length %lld != local state size %lld", n, need);
    if (nk_buffers(need)) return 1;
    CK(cudaMemcpyAsync(g.nkU, U, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (nk_vec_kernel(g.nkU, nullptr, nullptr, 0.0, 0)) return 1;
    if (adfb_residual(1, kNkFlags)) return 1;
    if (nk_vec_kernel(nullptr, nullptr, g.nkF0, 1.0, 2)) return 1;
    double uu = 0.0;
    if (nk_sumsq(g.nkU, need, &uu)) return 1;
    g.nkUnorm = sqrt(uu);
    g.nkHaveBase = true;
    g.ankHaveBase = false; g.ankTurbHaveBase = false;   // the ANK bases share the buffers
    return 0;
}

// MatMult of the MFFD shell: y = (F(U + h a) - F(U)) / h.  h > 0: use it as given;
// h <= 0: PETSc's default Walker-Pernice choice h = error_rel * sqrt(1 + ||U||) / ||a||
// with error_rel = sqrt(machine epsilon) (PARITY UNPINNED at this boundary, see DESIGN.md).
// y = (F(U + h a) - F(U)) / h with a in g.nkA, y into g.nkY (device); returns 2 when a == 0 (y = 0, no residual)
static int mffd_core(long long need, double h) {
    if (h <= 0.0) {
        double aa = 0.0;
        if (nk_sumsq(g.nkA, need, &aa)) return 1;
        if (aa == 0.0) {
            g.nkLastH = 0.0;
            return 2;
        }
        h = 1.4901161193847656e-08 * sqrt(1.0 + g.nkUnorm) / sqrt(aa);
    }
    g.nkLastH = h;
    // fused form (NKSolvers.F90:437-461 in one pass each way): the perturbation is formed together with p / rlv / rev of
    // the owned cells, and the kernels that write dw (tile kernel, k_sa) form y = (R - F0) / h of their rows; bitwise
    // the unfused product (same operations on the same operands).  ADFB_MFFD_FUSED=0, or a block the tile kernel does not
    // take (matrix / upwind dissipation, coarse level), selects the three-pass form.
    // The two extra vector passes of the three-pass form cost less than the strided AoS accesses of the epilogue inside
    // the tile kernel (the product is not bandwidth bound), so the three-pass form stays the default; ADFB_MFFD_FUSED=1
    // selects the fused one.
    bool fuse = false;
    { const char* e = getenv("ADFB_MFFD_FUSED"); if (e && e[0] == '1') fuse = true; }
    if (g_kt.on) fuse = false;
    for (Block& b : g.blocks)
        if (b.alive && b.level == 1 && !tile_kernel_applies(b.d, b.dev, residual_discr(1, true))) fuse = false;
    if (overset_present(1)) fuse = false;   // the exchange rewrites owned fringe cells: p, rhoE must follow (k_etot_owned)
    if (fuse) {
        if (!g.dMffd) {
            CK(cudaMalloc((void**)&g.dMffd, sizeof(MffdDev)));
            CK(cudaMallocHost((void**)&g.hMffd, sizeof(MffdDev)));
        }
        int nw0 = 6;
        for (Block& b : g.blocks) if (b.alive && b.level == 1) { nw0 = b.nw; break; }
        g.hMffd->F0 = g.nkF0; g.hMffd->y = g.nkY; g.hMffd->h = h; g.hMffd->nw = nw0;
        CK(cudaMemcpyAsync(g.dMffd, g.hMffd, sizeof(MffdDev), cudaMemcpyHostToDevice, g.stream));
        long long off = 0;
        for (Block& b : g.blocks) {
            if (!b.alive || b.level != 1) continue;
            const long long nc = (long long)b.d.nx * b.d.ny * b.d.nz;
            KT_BEGIN(K_MFFD, g.stream);
            k_nkvec_prep<<<(unsigned)((nc + 255) / 256), 256, 0, g.stream>>>(b.d, b.dev, b.nw, g.nkA + off, g.nkU + off, g.dMffd, 1);
            KT_END(K_MFFD, g.stream);
            off += nc * b.nw;
        }
        g.mffdFuse = true;
        const int rc = adfb_residual(1, kNkFlags);
        g.mffdFuse = false;
        return rc ? 1 : 0;
    }
    if (nk_vec_kernel(g.nkA, g.nkU, nullptr, h, 1)) return 1;
    if (adfb_residual(1, kNkFlags)) return 1;
    if (nk_vec_kernel(nullptr, g.nkF0, g.nkY, h, 3)) return 1;
    return 0;
}
int adfb_mffd_apply(const double* a, double* y, long long n, double h) {
    ADFB_RANGE("adfb_mffd_apply");
    NEED_INIT();
    if (!g.nkHaveBase) return fail("adfb_mffd_apply: adfb_mffd_set_base has not been called");
    const long long need = adfb_state_size();
    if (!a || !y || n != need || (size_t)need > g.nkN) return fail("adfb_mffd_apply: vector length %lld != local state size %lld", n, need);
    CK(cudaMemcpyAsync(g.nkA, a, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    const int rc = mffd_core(need, h);
    if (rc == 1) return 1;
    if (rc == 2) {
        CK(cudaStreamSynchronize(g.stream));
        memset(y, 0, need * sizeof(double));
        return 0;
    }
    CK(cudaMemcpyAsync(y, g.nkY, need * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
// the same product for Krylov vectors that already live on THIS device (PETSc VECCUDA: VecCUDAGetArrayRead /
// VecCUDAGetArrayWrite): no PCIe traffic; the result is complete when the call returns
int adfb_mffd_apply_device(const double* aDev, double* yDev, long long n, double h) {
    ADFB_RANGE("adfb_mffd_apply_device");
    NEED_INIT();
    if (!g.nkHaveBase) return fail("adfb_mffd_apply_device: adfb_mffd_set_base has not been called");
    const long long need = adfb_state_size();
    if (!aDev || !yDev || n != need || (size_t)need > g.nkN)
        return fail("adfb_mffd_apply_device: vector length %lld != local state size %lld", n, need);
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, aDev) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != g.device)
        return fail("adfb_mffd_apply_device: a is not a device pointer of device %d", g.device);
    if (cudaPointerGetAttributes(&at, yDev) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != g.device)
        return fail("adfb_mffd_apply_device: y is not a device pointer of device %d", g.device);
    CK(cudaMemcpyAsync(g.nkA, aDev, need * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    const int rc = mffd_core(need, h);
    if (rc == 1) return 1;
    if (rc == 2) CK(cudaMemsetAsync(yDev, 0, need * sizeof(double), g.stream));
    else CK(cudaMemcpyAsync(yDev, g.nkY, need * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
double adfb_mffd_last_h(void) { return g.nkLastH; }

// referenceShockSensor, src/adjoint/adjointUtils.F90:1900-1950
int adfb_reference_shock_sensor(int level) {
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_reference_shock_sensor: adfb_set_params has not been called");
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        KT_BEGIN(K_MISC, g.stream);
        k_shock<<<(unsigned)((b.d.N + 255) / 256), 256, 0, g.stream>>>(b.d, b.dev, residual_discr(level, true));
        KT_END(K_MISC, g.stream);
    }
    CK(cudaGetLastError());
    return 0;
}

// applyAllBC (+ turbulence halos), src/solver/BCRoutines.F90:57, turbBCRoutines.F90:49
int adfb_apply_bcs(int level, int secondHalo, int withTurb) {
    ADFB_RANGE("adfb_apply_bcs");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_apply_bcs: adfb_set_params has not been called");
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        if (launch_bc_levels(b.d, b.dev, b.subfaces, secondHalo, withTurb && g.prm.equations == ADFB_RANS, 1, g.stream)) return fail("BC launch failed");
    }
    return 0;
}

// timeStep(onlyRadii), src/solver/solverUtils.F90:43-355 (timeStep_block).  The radii are needed only when the residual of
// the level reads them, i.e. with scalar dissipation: spaceDiscr up to the ground level, spaceDiscrCoarse above it
// (radiiNeededFine / radiiNeededCoarse, inputParamRoutines.F90:2829-2833).  Otherwise an only-radii call returns at once and
// leaves the radii of the last full call; the residual of a coarse ground level with fine = matrix or upwind and coarse =
// scalar reads exactly those.  dirScaling is off unless spaceDiscr is scalar dissipation (:2824).
int adfb_timestep(int level, int onlyRadii) {
    ADFB_RANGE("adfb_timestep");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_timestep: adfb_set_params has not been called");
    const bool above = above_ground(level);
    const bool radiiNeeded = (above ? g.prm.spaceDiscrCoarse : g.prm.spaceDiscr) == ADFB_DISS_SCALAR;
    if (onlyRadii && !radiiNeeded) return 0;
    const int scaleRad = !above && g.prm.spaceDiscr == ADFB_DISS_SCALAR;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        dim3 tb(32, 4, 2);
        dim3 gr((b.d.NI + 31) / 32, (b.d.NJ + 3) / 4, (b.d.NK + 1) / 2);
        KT_BEGIN(K_PREP, g.stream);
        launch_pdl(k_prep, gr, tb, g.stream, b.d, b.dev, onlyRadii ? 0 : 1, 1, 0, INT_MAX, residual_discr(level, false), scaleRad);
        KT_END(K_PREP, g.stream);
    }
    CK(cudaGetLastError());
    return 0;
}

static void launch_mg_cells1(const Dims& d, const BlockDev& b, int mode, cudaStream_t s);
// `initres(1,nwf); sourceTerms; residual` of the smoother loops (smoothers.F90:73-75,
// multiGrid.F90:883-888): mean-flow residual with rFil = cdisRK(rkStage+1), fw persistent.
static int adfb_smoother_residual_body(int level, int rkStage) {
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_smoother_residual: adfb_set_params has not been called");
    if (rkStage < 0 || rkStage > 5) return fail("adfb_smoother_residual: rkStage %d out of range", rkStage);
    const double rFil = g.prm.cdisRK[rkStage];
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        // coarse level: initRes starts from the residual forcing term (dw = wr)
        if (launch_residual_core(b.d, b.dev, g.prm, g.env, residual_discr(level, false), ADFB_RES_FLOW, rFil, 1, 0, g.stream,
                                 above_ground(level) ? g.mgInitWr : 0))
            return fail("residual launch failed");
        // the primitive <-> conservative round trip that inviscidDissFluxScalarCoarse leaves on w (the matrix form does not convert)
        if (above_ground(level) && fabs(rFil) >= 1.e-10 && g.prm.spaceDiscrCoarse == ADFB_DISS_SCALAR) launch_mg_cells1(b.d, b.dev, 2, g.stream);
    }
    CK(cudaGetLastError());
    return 0;
}
int adfb_smoother_residual(int level, int rkStage) {
    ADFB_RANGE("adfb_smoother_residual");
    NEED_INIT();
    const unsigned long long key = (3ull << 40) | ((unsigned long long)level << 32) | ((unsigned)g.mgInitWr << 8) | (unsigned)rkStage;
    return run_graphed(key, [&]() { return adfb_smoother_residual_body(level, rkStage); });
}

// executeRkStage, src/solver/smoothers.F90:90-382
static int adfb_rk_stage_body(int level, int rkStage) {
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_rk_stage: adfb_set_params has not been called");
    if (rkStage < 1 || rkStage > g.prm.nRKStages) return fail("adfb_rk_stage: stage %d out of 1..%d", rkStage, g.prm.nRKStages);
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        // currentCfl = cflCoarse unless currentLevel == 1; second halos only on the ground level (smoothers.F90:131-140)
        AdfbParams prmL = g.prm;
        if (level > 1) prmL.cfl = g.prm.cflCoarse;
        if (launch_rk_update(b.d, b.dev, prmL, g.env, rkStage, g.stream, above_ground(level) ? 5 : 0)) return fail("RK update launch failed");
    }
    // whalo2(level, 1, nwf, T, T, T) / whalo1 on coarse levels (the pattern of the level holds the matching lists):
    // the trailing computeEtotBlock is idempotent here unless an overset pattern interpolates into fringe cells.
    // Multi-rank: the updated owned cells travel while the BC chain runs.
    const bool split = halo_split_ok(level);
    if (split && halo_exchange_impl(level, 1, 5, 1, 1, overset_present(level), 1)) return 1;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        if (launch_bc_levels(b.d, b.dev, b.subfaces, above_ground(level) ? 0 : 1, 0, 1, g.stream)) return fail("flow BC launch failed");
    }
    if (halo_exchange_impl(level, 1, 5, 1, 1, overset_present(level), split ? 2 : 0)) return 1;
    CK(cudaGetLastError());
    return 0;
}
int adfb_rk_stage(int level, int rkStage) {
    ADFB_RANGE("adfb_rk_stage");
    NEED_INIT();
    const unsigned long long key = (2ull << 40) | ((unsigned long long)level << 32) | (unsigned)rkStage;
    return run_graphed(key, [&]() { return adfb_rk_stage_body(level, rkStage); });
}

// executeDADIStep, src/solver/smoothers.F90:425-693
static int adfb_dadi_step_body(int level) {
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_dadi_step: adfb_set_params has not been called");
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        AdfbParams prmL = g.prm;   // coarse levels: cflCoarse, first halos only, frozen eddy viscosity (smoothers.F90:463-472)
        if (level > 1) prmL.cfl = g.prm.cflCoarse;
        if (launch_dadi(b.d, b.dev, prmL, g.stream)) return fail("DADI launch failed");
        if (launch_dadi_update(b.d, b.dev, prmL, g.env, g.stream, above_ground(level) ? 5 : 0)) return fail("DADI update launch failed");
        if (launch_bc_levels(b.d, b.dev, b.subfaces, above_ground(level) ? 0 : 1, 0, 1, g.stream)) return fail("flow BC launch failed");
    }
    if (halo_exchange_impl(level, 1, 5, 1, 1, overset_present(level))) return 1;
    CK(cudaGetLastError());
    return 0;
}
int adfb_dadi_step(int level) {
    ADFB_RANGE("adfb_dadi_step");
    NEED_INIT();
    const unsigned long long key = (4ull << 40) | ((unsigned long long)level << 32);
    return run_graphed(key, [&]() { return adfb_dadi_step_body(level); });
}

// DADISmoother, src/solver/smoothers.F90:383-421
static int adfb_dadi_cycle_body(int level, int nSubiterations) {
    NEED_INIT();
    if (nSubiterations < 1) return fail("adfb_dadi_cycle: nSubiterations must be >= 1");
    for (int sub = 1; sub <= nSubiterations - 1; sub++) {
        if (adfb_dadi_step(level)) return 1;
        if (adfb_smoother_residual(level, 0)) return 1;
    }
    return adfb_dadi_step(level);
}
int adfb_dadi_cycle(int level, int nSubiterations) {
    ADFB_RANGE("adfb_dadi_cycle");
    NEED_INIT();
    const unsigned long long key = (7ull << 40) | ((unsigned long long)level << 32) | (unsigned)nSubiterations;
    return run_graphed(key, [&]() { return adfb_dadi_cycle_body(level, nSubiterations); });
}

// turbSolveDDADI, src/turbulence/turbAPI.F90:4-95 (Spalart-Allmaras)
static int adfb_sa_ddadi_body(int level, int nSubIterTurb) {
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_sa_ddadi: adfb_set_params has not been called");
    if (g.prm.equations != ADFB_RANS) return fail("adfb_sa_ddadi: equations are not RANS");
    if (nSubIterTurb < 1) return fail("adfb_sa_ddadi: nSubIterTurb must be >= 1");
    for (int iter = 0; iter < nSubIterTurb; iter++) {
        for (Block& b : g.blocks) {
            if (!b.alive || b.level != level) continue;
            if (launch_sa_block(b.d, b.dev, g.prm, b.subfaces, g.stream)) return fail("SA DD-ADI launch failed");
        }
        // whalo2(groundLevel, nt1, nt2, .false., .false., .true.), turbAPI.F90:91
        if (halo_exchange_impl(level, 6, 6, 0, 1, false)) return 1;
    }
    CK(cudaGetLastError());
    return 0;
}
int adfb_sa_ddadi(int level, int nSubIterTurb) {
    ADFB_RANGE("adfb_sa_ddadi");
    NEED_INIT();
    const unsigned long long key = (5ull << 40) | ((unsigned long long)level << 32) | (unsigned)nSubIterTurb;
    return run_graphed(key, [&]() { return adfb_sa_ddadi_body(level, nSubIterTurb); });
}

// RungeKuttaSmoother, src/solver/smoothers.F90:4-86
static int adfb_rk_cycle_body(int level) {
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_rk_cycle: adfb_set_params has not been called");
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        CK(cudaMemcpyAsync(b.dev.wn, b.dev.w, (size_t)b.d.N * 5 * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
        CK(cudaMemcpyAsync(b.dev.pn, b.dev.p, (size_t)b.d.N * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    }
    for (int st = 1; st <= g.prm.nRKStages - 1; st++) {
        if (adfb_rk_stage(level, st)) return 1;
        if (adfb_smoother_residual(level, st)) return 1;
    }
    return adfb_rk_stage(level, g.prm.nRKStages);
}
int adfb_rk_cycle(int level) {
    ADFB_RANGE("adfb_rk_cycle");
    NEED_INIT();
    const unsigned long long key = (6ull << 40) | ((unsigned long long)level << 32);
    return run_graphed(key, [&]() { return adfb_rk_cycle_body(level); });
}


// ---------------------------------------------------------------------------
// ANK pieces (module ANKSolver, src/NKSolver/NKSolvers.F90)
static int ank_nstate(const Block& b) { return g.ank.coupled ? b.nw : 5; }
static long long ank_vec_size(void) {
    long long n = 0;
    for (Block& b : g.blocks)
        if (b.alive && b.level == 1) n += (long long)b.d.nx * b.d.ny * b.d.nz * ank_nstate(b);
    return n;
}
static unsigned ank_res_flags(void) {
    unsigned f = ADFB_RES_FLOW;
    if (g.ank.useDissApprox) f |= ADFB_RES_DISS_APPROX;
    if (!g.ank.useFullVisc && g.ank.useDissApprox) f |= ADFB_RES_VISC_APPROX;   // :2489
    if (g.ank.coupled) f |= ADFB_RES_TURB;
    return f;
}
int adfb_ank_set_params(const AdfbAnkParams* ank) {
    NEED_INIT();
    if (!ank) return fail("adfb_ank_set_params: null");
    if (!(ank->cfl > 0.0) || !(ank->cflLimit > 0.0) || !(ank->turbCFLScale > 0.0)) return fail("adfb_ank_set_params: CFL values must be positive");
    if (ank->charTimeStepType < 0 || ank->charTimeStepType > 2) return fail("adfb_ank_set_params: charTimeStepType %d (0 None, 1 VLR, 2 Turkel)", ank->charTimeStepType);
    if (ank->coupled && g.havePrm && g.prm.equations != ADFB_RANS) return fail("adfb_ank_set_params: coupled ANK needs the RANS equations");
    // No drop_graphs: the ANK products launch their own kernels with g.ank as an argument at every call, and the residual
    // they call is keyed by its flags, which carry the ANK options it depends on (ank_res_flags).
    g.ank = *ank;
    g.haveAnk = true; g.ankHaveT = false; g.ankHaveBase = false;
    return 0;
}
int adfb_ank_time_step_mat(void) {
    ADFB_RANGE("adfb_ank_time_step_mat");
    NEED_INIT();
    if (!g.havePrm || !g.haveAnk) return fail("adfb_ank_time_step_mat: adfb_set_params / adfb_ank_set_params have not been called");
    size_t need = 0;
    for (Block& b : g.blocks)
        if (b.alive && b.level == 1) need += (size_t)b.d.nx * b.d.ny * b.d.nz * ank_nstate(b) * ank_nstate(b);
    if (g.ankTN < need) {
        if (g.ankT) cudaFree(g.ankT);
        g.ankT = nullptr; g.ankTN = 0;
        CK(cudaMalloc((void**)&g.ankT, need * sizeof(double)));
        g.ankTN = need;
    }
    size_t off = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        const long long nc = (long long)b.d.nx * b.d.ny * b.d.nz;
        const int ns = ank_nstate(b);
        KT_BEGIN(K_MFFD, g.stream);
        if (ns == 5) k_ank_tsblock<5><<<(unsigned)((nc + 63) / 64), 64, 0, g.stream>>>(b.d, b.dev, g.ank, g.ankT + off);
        else k_ank_tsblock<6><<<(unsigned)((nc + 63) / 64), 64, 0, g.stream>>>(b.d, b.dev, g.ank, g.ankT + off);
        KT_END(K_MFFD, g.stream);
        off += (size_t)nc * ns * ns;
    }
    CK(cudaGetLastError());
    g.ankHaveT = true;
    return 0;
}
static int ank_vec_kernel(const double* vec, const double* base, double* out, double* pert, double h, int mode) {
    long long off = 0;
    size_t offT = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        const int ns = ank_nstate(b);
        const long long nc = (long long)b.d.nx * b.d.ny * b.d.nz, n = nc * ns;
        KT_BEGIN(K_MFFD, g.stream);
        k_ankvec<<<(unsigned)((n + 255) / 256), 256, 0, g.stream>>>(b.d, b.dev, ns, vec ? vec + off : nullptr, base ? base + off : nullptr,
                                                                    out ? out + off : nullptr, pert ? pert + off : nullptr,
                                                                    g.ankT ? g.ankT + offT : nullptr, h, mode);
        KT_END(K_MFFD, g.stream);
        off += n;
        offT += (size_t)nc * ns * ns;
    }
    CK(cudaGetLastError());
    return 0;
}
static int ank_ready(const char* who, long long n, long long* need) {
    if (!g.havePrm || !g.haveAnk) return fail("%s: adfb_set_params / adfb_ank_set_params have not been called", who);
    if (!g.ankHaveT) return fail("%s: adfb_ank_time_step_mat has not been called", who);
    *need = ank_vec_size();
    if (n != *need) return fail("%s: vector length %lld != %lld (nState entries per owned cell)", who, n, *need);
    if (nk_buffers(adfb_state_size())) return 1;
    if (g.ankPertN < (size_t)*need) {
        if (g.ankPert) cudaFree(g.ankPert);
        g.ankPert = nullptr; g.ankPertN = 0;
        CK(cudaMalloc((void**)&g.ankPert, *need * sizeof(double)));
        g.ankPertN = *need;
    }
    return 0;
}
// FormFunction_mf (:2468-2538)
int adfb_ank_form_function(const double* inVec, double* rVec, long long n) {
    ADFB_RANGE("adfb_ank_form_function");
    NEED_INIT();
    long long need = 0;
    if (!inVec || !rVec) return fail("adfb_ank_form_function: null vector");
    if (ank_ready("adfb_ank_form_function", n, &need)) return 1;
    CK(cudaMemcpyAsync(g.nkA, inVec, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (ank_vec_kernel(g.nkA, nullptr, nullptr, nullptr, 0.0, 0)) return 1;
    if (adfb_residual(1, ank_res_flags())) return 1;
    if (ank_vec_kernel(g.nkA, nullptr, g.nkY, nullptr, 1.0, 2)) return 1;
    CK(cudaMemcpyAsync(rVec, g.nkY, need * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
int adfb_ank_mffd_set_base(const double* U, long long n) {
    NEED_INIT();
    long long need = 0;
    if (!U) return fail("adfb_ank_mffd_set_base: null vector");
    if (ank_ready("adfb_ank_mffd_set_base", n, &need)) return 1;
    CK(cudaMemcpyAsync(g.nkU, U, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (ank_vec_kernel(g.nkU, nullptr, nullptr, nullptr, 0.0, 0)) return 1;
    if (adfb_residual(1, ank_res_flags())) return 1;
    if (ank_vec_kernel(g.nkU, nullptr, g.nkF0, nullptr, 1.0, 2)) return 1;
    double uu = 0.0;
    if (nk_sumsq(g.nkU, need, &uu)) return 1;
    g.ankUnorm = sqrt(uu);
    g.ankHaveBase = true;
    g.nkHaveBase = false; g.ankTurbHaveBase = false;   // the NK base shares the buffers
    return 0;
}
// y = (F(U + h a) - F(U)) / h with a in g.nkA, y into g.nkY; returns 2 when a == 0
static int ank_mffd_core(long long need, double h) {
    if (h <= 0.0) {
        double aa = 0.0;
        if (nk_sumsq(g.nkA, need, &aa)) return 1;
        if (aa == 0.0) { g.nkLastH = 0.0; return 2; }
        h = 1.4901161193847656e-08 * sqrt(1.0 + g.ankUnorm) / sqrt(aa);
    }
    g.nkLastH = h;
    if (ank_vec_kernel(g.nkA, g.nkU, nullptr, g.ankPert, h, 1)) return 1;
    if (adfb_residual(1, ank_res_flags())) return 1;
    if (ank_vec_kernel(g.ankPert, g.nkF0, g.nkY, nullptr, h, 3)) return 1;
    return 0;
}
int adfb_ank_mffd_apply(const double* a, double* y, long long n, double h) {
    ADFB_RANGE("adfb_ank_mffd_apply");
    NEED_INIT();
    long long need = 0;
    if (!a || !y) return fail("adfb_ank_mffd_apply: null vector");
    if (ank_ready("adfb_ank_mffd_apply", n, &need)) return 1;
    if (!g.ankHaveBase) return fail("adfb_ank_mffd_apply: adfb_ank_mffd_set_base has not been called");
    CK(cudaMemcpyAsync(g.nkA, a, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    const int rc = ank_mffd_core(need, h);
    if (rc == 1) return 1;
    if (rc == 2) { CK(cudaStreamSynchronize(g.stream)); memset(y, 0, need * sizeof(double)); return 0; }
    CK(cudaMemcpyAsync(y, g.nkY, need * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
// the same product for Krylov vectors resident on this device (PETSc VECCUDA), like adfb_mffd_apply_device
int adfb_ank_mffd_apply_device(const double* aDev, double* yDev, long long n, double h) {
    ADFB_RANGE("adfb_ank_mffd_apply_device");
    NEED_INIT();
    long long need = 0;
    if (!aDev || !yDev) return fail("adfb_ank_mffd_apply_device: null vector");
    if (ank_ready("adfb_ank_mffd_apply_device", n, &need)) return 1;
    if (!g.ankHaveBase) return fail("adfb_ank_mffd_apply_device: adfb_ank_mffd_set_base has not been called");
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, aDev) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != g.device)
        return fail("adfb_ank_mffd_apply_device: a is not a device pointer of device %d", g.device);
    if (cudaPointerGetAttributes(&at, yDev) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != g.device)
        return fail("adfb_ank_mffd_apply_device: y is not a device pointer of device %d", g.device);
    CK(cudaMemcpyAsync(g.nkA, aDev, need * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    const int rc = ank_mffd_core(need, h);
    if (rc == 1) return 1;
    if (rc == 2) CK(cudaMemsetAsync(yDev, 0, need * sizeof(double), g.stream));
    else CK(cudaMemcpyAsync(yDev, g.nkY, need * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
// physicalityCheckANK (:3013-3210)
// ---- turbulence KSP of the decoupled ANK (ANKTurbSolveKSP, NKSolvers.F90:3337 ff.): one turbulence variable per owned cell
static long long ank_turb_vec_size(void) {
    long long n = 0;
    for (Block& b : g.blocks)
        if (b.alive && b.level == 1) n += (long long)b.d.nx * b.d.ny * b.d.nz;
    return n;
}
static int ank_turb_ready(const char* who, long long n) {
    if (!g.havePrm || !g.haveAnk) return fail("%s: adfb_set_params / adfb_ank_set_params have not been called", who);
    if (g.prm.equations != ADFB_RANS) return fail("%s: needs the RANS equations (a turbulence variable)", who);
    const long long need = ank_turb_vec_size();
    if (n != need) return fail("%s: vector length %lld != %lld (one turbulence variable per owned cell)", who, n, need);
    if (nk_buffers(adfb_state_size())) return 1;
    if (g.ankPertN < (size_t)need) {
        if (g.ankPert) cudaFree(g.ankPert);
        g.ankPert = nullptr; g.ankPertN = 0;
        CK(cudaMalloc((void**)&g.ankPert, need * sizeof(double)));
        g.ankPertN = need;
    }
    return 0;
}
// blocketteRes without useUpdateIntermed leaves the block's dtl alone (the tile's time step stays local, blockette.F90:1929),
// the device residual always stores it: the time-stepping term uses the copy taken before the residual (work array 0)
static int ank_turb_save_dtl(void) {
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        CK(cudaMemcpyAsync(b.dev.scratch, b.dev.dtl, (size_t)b.d.N * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    }
    return 0;
}
static int ank_turb_vec_kernel(const double* vec, const double* base, double* out, double* pert, double h, int mode) {
    long long off = 0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        const long long nc = (long long)b.d.nx * b.d.ny * b.d.nz;
        KT_BEGIN(K_MFFD, g.stream);
        k_ankvec_turb<<<(unsigned)((nc + 255) / 256), 256, 0, g.stream>>>(b.d, b.dev, g.ank, b.dev.scratch, vec ? vec + off : nullptr, base ? base + off : nullptr,
                                                                         out ? out + off : nullptr, pert ? pert + off : nullptr, h, mode);
        KT_END(K_MFFD, g.stream);
        off += nc;
    }
    CK(cudaGetLastError());
    return 0;
}
// FormFunction_mf_turb (:2540-2612): setWANK(inVec, nt1, nt2); blocketteRes(useFlowRes = .false.); setRVecANKTurb; time-stepping term
int adfb_ank_form_function_turb(const double* inVec, double* rVec, long long n) {
    ADFB_RANGE("adfb_ank_form_function_turb");
    NEED_INIT();
    if (!inVec || !rVec) return fail("adfb_ank_form_function_turb: null vector");
    if (ank_turb_ready("adfb_ank_form_function_turb", n)) return 1;
    CK(cudaMemcpyAsync(g.nkA, inVec, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (ank_turb_save_dtl()) return 1;
    if (ank_turb_vec_kernel(g.nkA, nullptr, nullptr, nullptr, 0.0, 0)) return 1;
    if (adfb_residual(1, ADFB_RES_TURB)) return 1;
    if (ank_turb_vec_kernel(g.nkA, nullptr, g.nkY, nullptr, 1.0, 2)) return 1;
    CK(cudaMemcpyAsync(rVec, g.nkY, n * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
// the matrix-free product of the turbulence KSP (MatMFFD shell over FormFunction_mf_turb): base state, then
// y = (F(U + h a) - F(U)) / h with a given h > 0
int adfb_ank_mffd_turb_set_base(const double* U, long long n) {
    ADFB_RANGE("adfb_ank_mffd_turb_set_base");
    NEED_INIT();
    if (!U) return fail("adfb_ank_mffd_turb_set_base: null vector");
    if (ank_turb_ready("adfb_ank_mffd_turb_set_base", n)) return 1;
    g.nkHaveBase = false; g.ankHaveBase = false;   // the NK / ANK bases share the buffers
    CK(cudaMemcpyAsync(g.nkU, U, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (ank_turb_save_dtl()) return 1;
    if (ank_turb_vec_kernel(g.nkU, nullptr, nullptr, nullptr, 0.0, 0)) return 1;
    if (adfb_residual(1, ADFB_RES_TURB)) return 1;
    if (ank_turb_vec_kernel(g.nkU, nullptr, g.nkF0, nullptr, 1.0, 2)) return 1;
    CK(cudaStreamSynchronize(g.stream));
    g.ankTurbHaveBase = true;
    return 0;
}
int adfb_ank_mffd_turb_apply(const double* a, double* y, long long n, double h) {
    ADFB_RANGE("adfb_ank_mffd_turb_apply");
    NEED_INIT();
    if (!a || !y) return fail("adfb_ank_mffd_turb_apply: null vector");
    if (!(h > 0.0)) return fail("adfb_ank_mffd_turb_apply: h must be positive");
    if (ank_turb_ready("adfb_ank_mffd_turb_apply", n)) return 1;
    if (!g.ankTurbHaveBase || g.nkHaveBase || g.ankHaveBase) return fail("adfb_ank_mffd_turb_apply: adfb_ank_mffd_turb_set_base has not been called");
    CK(cudaMemcpyAsync(g.nkA, a, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    if (ank_turb_vec_kernel(g.nkA, g.nkU, nullptr, g.ankPert, h, 1)) return 1;
    if (adfb_residual(1, ADFB_RES_TURB)) return 1;
    if (ank_turb_vec_kernel(g.ankPert, g.nkF0, g.nkY, nullptr, h, 3)) return 1;
    CK(cudaMemcpyAsync(y, g.nkY, n * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    return 0;
}
// physicalityCheckANKTurb (:3212-3335)
int adfb_ank_physicality_check_turb(const double* wVec, double* deltaW, long long n, double* lambdaP) {
    ADFB_RANGE("adfb_ank_physicality_check_turb");
    NEED_INIT();
    if (!wVec || !deltaW || !lambdaP) return fail("adfb_ank_physicality_check_turb: null argument");
    if (ank_turb_ready("adfb_ank_physicality_check_turb", n)) return 1;
    CK(cudaMemcpyAsync(g.nkA, wVec, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(g.nkY, deltaW, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    const int nPart = 512;
    KT_BEGIN(K_MFFD, g.stream);
    k_ank_phys_turb<<<nPart, 256, 0, g.stream>>>(n, g.ank, g.nkA, g.nkY, *lambdaP, g.dRed);
    KT_END(K_MFFD, g.stream);
    KT_BEGIN(K_MFFD, g.stream);
    k_min_final<<<1, 256, 0, g.stream>>>(g.dRed, nPart);
    KT_END(K_MFFD, g.stream);
    if (g.nranks > 1) {
        const int rc = g.nccl.AllReduce(g.dRed + nPart, g.dRed + nPart, 1, kNcclDouble, kNcclMin, g.comm, g.stream);
        if (rc != 0) return fail("ncclAllReduce: %s", g.nccl.GetErrorString(rc));
    }
    CK(cudaMemcpyAsync(g.hRed, g.dRed + nPart, sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaMemcpyAsync(deltaW, g.nkY, n * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    CK(cudaGetLastError());
    *lambdaP = g.hRed[0];
    return 0;
}
int adfb_ank_physicality_check(const double* wVec, double* deltaW, long long n, double* lambdaP) {
    ADFB_RANGE("adfb_ank_physicality_check");
    NEED_INIT();
    if (!g.haveAnk) return fail("adfb_ank_physicality_check: adfb_ank_set_params has not been called");
    if (!wVec || !deltaW || !lambdaP) return fail("adfb_ank_physicality_check: null argument");
    const long long need = ank_vec_size();
    if (n != need) return fail("adfb_ank_physicality_check: vector length %lld != %lld", n, need);
    if (nk_buffers(adfb_state_size())) return 1;
    CK(cudaMemcpyAsync(g.nkA, wVec, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    CK(cudaMemcpyAsync(g.nkY, deltaW, need * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    int ns = 5;
    for (Block& b : g.blocks) if (b.alive && b.level == 1) { ns = ank_nstate(b); break; }
    const int nPart = 512;
    KT_BEGIN(K_MFFD, g.stream);
    k_ank_phys<<<nPart, 256, 0, g.stream>>>(need / ns, ns, g.ank.coupled, g.ank, g.nkA, g.nkY, *lambdaP, g.dRed);
    KT_END(K_MFFD, g.stream);
    KT_BEGIN(K_MFFD, g.stream);
    k_min_final<<<1, 256, 0, g.stream>>>(g.dRed, nPart);
    KT_END(K_MFFD, g.stream);
    if (g.nranks > 1) {
        const int rc = g.nccl.AllReduce(g.dRed + nPart, g.dRed + nPart, 1, kNcclDouble, kNcclMin, g.comm, g.stream);
        if (rc != 0) return fail("ncclAllReduce: %s", g.nccl.GetErrorString(rc));
    }
    CK(cudaMemcpyAsync(g.hRed, g.dRed + nPart, sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    if (g.ank.coupled) CK(cudaMemcpyAsync(deltaW, g.nkY, need * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    CK(cudaGetLastError());
    *lambdaP = g.hRed[0];
    return 0;
}

// ---------------------------------------------------------------------------
// multigrid (src/solver/multiGrid.F90)
static void launch_mg_cells1(const Dims& d, const BlockDev& b, int mode, cudaStream_t s) {
    dim3 tb(32, 4, 2);
    dim3 gr((d.ie + 31) / 32, (d.je + 3) / 4, (d.ke + 1) / 2);
    KT_BEGIN(K_MISC, s);
    launch_pdl(k_mg_cells1, gr, tb, s, d, b, mode);
    KT_END(K_MISC, s);
}

int adfb_block_set_mg(int coarseBlk, int fineBlk, const int32_t* mgIFine, const int32_t* mgJFine, const int32_t* mgKFine,
                      const double* mgIWeight, const double* mgJWeight, const double* mgKWeight, const int32_t* mgICoarse,
                      const int32_t* mgJCoarse, const int32_t* mgKCoarse) {
    NEED_INIT();
    drop_graphs();
    Block* c = get_block(coarseBlk);
    Block* f = get_block(fineBlk);
    if (!c || !f) return fail("adfb_block_set_mg: no block %d / %d", coarseBlk, fineBlk);
    if (c->level != f->level + 1) return fail("adfb_block_set_mg: block %d (level %d) is not one level coarser than block %d (level %d)",
                                              coarseBlk, c->level, fineBlk, f->level);
    if (!mgIFine || !mgJFine || !mgKFine || !mgIWeight || !mgJWeight || !mgKWeight || !mgICoarse || !mgJCoarse || !mgKCoarse)
        return fail("adfb_block_set_mg: all nine tables are required");
    // reference extents -> tables indexed by the Fortran index: mg?Fine(1:ie,2), mg?Weight(2:il), mg?Coarse(2:il_f,2)
    const int ce[3] = {c->d.ie, c->d.je, c->d.ke}, cl[3] = {c->d.il, c->d.jl, c->d.kl};
    const int fe[3] = {f->d.ie, f->d.je, f->d.ke}, fl[3] = {f->d.il, f->d.jl, f->d.kl};
    const int32_t* fin[3] = {mgIFine, mgJFine, mgKFine};
    const double* wgt[3] = {mgIWeight, mgJWeight, mgKWeight};
    const int32_t* coa[3] = {mgICoarse, mgJCoarse, mgKCoarse};
    for (void* q : c->mgAllocs) cudaFree(q);
    c->mgAllocs.clear();
    const int* dF[3]; const double* dW[3]; const int* dC[3];
    for (int a = 0; a < 3; a++) {
        std::vector<int> hf((size_t)(ce[a] + 1) * 2, 0), hc((size_t)(fe[a] + 1) * 2, 0);
        std::vector<double> hw((size_t)ce[a] + 1, 0.0);
        for (int m = 0; m < 2; m++)
            for (int i = 1; i <= ce[a]; i++) {
                const int v = fin[a][(i - 1) + ce[a] * m];
                if (v < 0 || v > fe[a] + 1) return fail("adfb_block_set_mg: mgFine entry %d out of the fine block", v);
                hf[i + (ce[a] + 1) * m] = v;
            }
        for (int i = 2; i <= cl[a]; i++) hw[i] = wgt[a][i - 2];
        for (int m = 0; m < 2; m++)
            for (int i = 2; i <= fl[a]; i++) {
                const int v = coa[a][(i - 2) + (fl[a] - 1) * m];
                if (v < 1 || v > ce[a]) return fail("adfb_block_set_mg: mgCoarse entry %d out of the coarse block (1:%d)", v, ce[a]);
                hc[i + (fe[a] + 1) * m] = v;
            }
        void *q1 = nullptr, *q2 = nullptr, *q3 = nullptr;
        CK(cudaMalloc(&q1, hf.size() * sizeof(int))); c->mgAllocs.push_back(q1);
        CK(cudaMalloc(&q2, hw.size() * sizeof(double))); c->mgAllocs.push_back(q2);
        CK(cudaMalloc(&q3, hc.size() * sizeof(int))); c->mgAllocs.push_back(q3);
        CK(cudaMemcpy(q1, hf.data(), hf.size() * sizeof(int), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(q2, hw.data(), hw.size() * sizeof(double), cudaMemcpyHostToDevice));
        CK(cudaMemcpy(q3, hc.data(), hc.size() * sizeof(int), cudaMemcpyHostToDevice));
        dF[a] = (const int*)q1; dW[a] = (const double*)q2; dC[a] = (const int*)q3;
    }
    c->mg.fI = dF[0]; c->mg.fJ = dF[1]; c->mg.fK = dF[2];
    c->mg.wI = dW[0]; c->mg.wJ = dW[1]; c->mg.wK = dW[2];
    c->mg.cI = dC[0]; c->mg.cJ = dC[1]; c->mg.cK = dC[2];
    c->fineBlk = fineBlk; f->coarseBlk = coarseBlk;
    return 0;
}

// transferToCoarseGrid, multiGrid.F90:5-324: from `fineLevel` to fineLevel + 1
static int adfb_mg_restrict_body(int fineLevel) {
    const int cl = fineLevel + 1;
    // fine residual: rkStage = 0; timeStep(.true.) = spectral radii only; initres; residual
    if (adfb_timestep(fineLevel, 1)) return 1;
    if (adfb_smoother_residual(fineLevel, 0)) return 1;
    bool any = false;
    for (Block& c : g.blocks) {
        if (!c.alive || c.level != cl) continue;
        if (c.fineBlk < 0) return fail("adfb_mg_restrict: block of level %d without adfb_block_set_mg", cl);
        if (!c.haveMetrics) return fail("adfb_mg_restrict: geometry of a coarse block was never set");
        Block& f = g.blocks[c.fineBlk];
        any = true;
        dim3 tb(32, 4, 1);
        dim3 gr((c.d.nx + 31) / 32, (c.d.ny + 3) / 4, c.d.nz);
        KT_BEGIN(K_MISC, g.stream);
        launch_pdl(k_mg_restrict, gr, tb, g.stream, c.d, c.dev, f.d, f.dev, c.mg);
        KT_END(K_MISC, g.stream);
        KT_BEGIN(K_MISC, g.stream);
        launch_pdl(k_mg_corner_rows, dim3(1), dim3(256), g.stream, c.d, c.dev);
        KT_END(K_MISC, g.stream);
        if (launch_bc_levels(c.d, c.dev, c.subfaces, 0, 0, 1, g.stream)) return fail("flow BC launch failed");
    }
    if (!any) return fail("adfb_mg_restrict: no blocks on level %d", cl);
    // whalo1(currentLevel, 1, nwf, T, T, T)
    if (halo_exchange_impl(cl, 1, 5, 1, 1, false)) return 1;
    if (adfb_timestep(cl, 0)) return 1;
    for (Block& c : g.blocks) {
        if (!c.alive || c.level != cl) continue;
        launch_mg_cells1(c.d, c.dev, 0, g.stream);
    }
    // residual of the restricted solution, started from zero, rFil = cdisRK(1)
    g.mgInitWr = 0;
    const int rc = adfb_smoother_residual(cl, 0);
    g.mgInitWr = 1;
    if (rc) return 1;
    for (Block& c : g.blocks) {
        if (!c.alive || c.level != cl) continue;
        dim3 tb(32, 4, 2);
        dim3 gr((c.d.nx + 31) / 32, (c.d.ny + 3) / 4, (c.d.nz + 1) / 2);
        KT_BEGIN(K_MISC, g.stream);
        launch_pdl(k_mg_forcing, gr, tb, g.stream, c.d, c.dev, g.prm.fcoll);
        KT_END(K_MISC, g.stream);
    }
    CK(cudaGetLastError());
    return 0;
}
int adfb_mg_restrict(int fineLevel) {
    ADFB_RANGE("adfb_mg_restrict");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_mg_restrict: adfb_set_params has not been called");
    const unsigned long long key = (8ull << 40) | ((unsigned long long)fineLevel << 32);
    return run_graphed(key, [&]() { return adfb_mg_restrict_body(fineLevel); });
}

// transferToFineGrid(corrections = .true.), multiGrid.F90:326-654: from fineLevel + 1 to `fineLevel`
static int adfb_mg_prolong_body(int fineLevel) {
    const int cl = fineLevel + 1;
    const double fact = g.prm.mgBoundCorr == 0 ? 0.0 : 1.0;
    for (Block& c : g.blocks) {
        if (!c.alive || c.level != cl) continue;
        if (c.fineBlk < 0) return fail("adfb_mg_prolong: block of level %d without adfb_block_set_mg", cl);
        Block& f = g.blocks[c.fineBlk];
        launch_mg_cells1(c.d, c.dev, 1, g.stream);
        for (const AdfbSubface& sf : c.subfaces) {   // setCorrectionsCoarseHalos: BCData order
            FaceDev fd = make_face(c.d, sf);
            dim3 tb(32, 4);
            dim3 gr((fd.icEnd - fd.icBeg + 1 + 31) / 32, (fd.jcEnd - fd.jcBeg + 1 + 3) / 4);
            KT_BEGIN(K_BC, g.stream);
            launch_pdl(k_mg_corr_halos, gr, tb, g.stream, c.d, c.dev, fd, fact, 5);
            KT_END(K_BC, g.stream);
        }
        dim3 tb(32, 4, 1);
        dim3 gr((f.d.nx + 31) / 32, (f.d.ny + 3) / 4, f.d.nz);
        KT_BEGIN(K_MISC, g.stream);
        launch_pdl(k_mg_prolong, gr, tb, g.stream, f.d, f.dev, c.d, c.dev, c.mg, f.nw);
        KT_END(K_MISC, g.stream);
        // applyAllBC(secondHalo): second halos on the ground level only
        if (launch_bc_levels(f.d, f.dev, f.subfaces, above_ground(fineLevel) ? 0 : 1, 0, 1, g.stream)) return fail("flow BC launch failed");
    }
    if (halo_exchange_impl(fineLevel, 1, 5, 1, 1, overset_present(fineLevel))) return 1;
    CK(cudaGetLastError());
    return 0;
}
int adfb_mg_prolong(int fineLevel) {
    ADFB_RANGE("adfb_mg_prolong");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_mg_prolong: adfb_set_params has not been called");
    const unsigned long long key = (9ull << 40) | ((unsigned long long)fineLevel << 32);
    return run_graphed(key, [&]() { return adfb_mg_prolong_body(fineLevel); });
}

// iteration%groundLevel of the solver loop `do groundLevel = mgStartlevel, 1, -1` (solvers.F90:63): the finest level of the
// multigrid cycles that follow.  Levels above it take the coarse-level branches; the ground level itself runs the fine-grid
// routines with cflCoarse (currentLevel /= 1), in the discretisation residual_discr picks for the entry point.
int adfb_set_ground_level(int level) {
    ADFB_RANGE("adfb_set_ground_level");
    NEED_INIT();
    if (level < 1) return fail("adfb_set_ground_level: level %d", level);
    bool have = false;
    for (Block& b : g.blocks) if (b.alive && b.level == level) have = true;
    if (!have) return fail("adfb_set_ground_level: no block of level %d", level);
    CK(cudaStreamSynchronize(g.stream));
    g.groundLevel = level;
    for (Block& b : g.blocks) if (b.alive) b.dev.coarse = b.level > level ? 1 : 0;
    drop_graphs();
    return 0;
}
int adfb_get_ground_level(void) { return g.groundLevel; }

// transferToFineGrid(corrections = .false.), multiGrid.F90:326-654, the step of the full-multigrid start-up that follows the
// cycles on ground level fineLevel + 1 (solvers.F90:83-95): the coarse SOLUTION (all nw variables, pressure in place of
// rho*E, boundary halos by setCorrectionsCoarseHalos with fact = 1) interpolated to the owned cells of `fineLevel`, halos
// by constant extrapolation (extrapolateSolution / extrapolateViscosities), turbulence BCs, flow BCs twice, exchange, flow
// BCs, exchange -- all with second halos (currentLevel < groundLevel).  The caller lowers the ground level afterwards.
static int adfb_mg_prolong_solution_body(int fineLevel) {
    const int cl = fineLevel + 1;
    for (Block& c : g.blocks) {
        if (!c.alive || c.level != cl) continue;
        if (c.fineBlk < 0) return fail("adfb_mg_prolong_solution: block of level %d without adfb_block_set_mg", cl);
        Block& f = g.blocks[c.fineBlk];
        if (c.nw != f.nw) return fail("adfb_mg_prolong_solution: coarse and fine block carry %d / %d variables", c.nw, f.nw);
        launch_mg_cells1(c.d, c.dev, 3, g.stream);
        for (const AdfbSubface& sf : c.subfaces) {   // setCorrectionsCoarseHalos: BCData order
            FaceDev fd = make_face(c.d, sf);
            dim3 tb(32, 4);
            dim3 gr((fd.icEnd - fd.icBeg + 1 + 31) / 32, (fd.jcEnd - fd.jcBeg + 1 + 3) / 4);
            KT_BEGIN(K_BC, g.stream);
            launch_pdl(k_mg_corr_halos, gr, tb, g.stream, c.d, c.dev, fd, 1.0, f.nw);
            KT_END(K_BC, g.stream);
        }
        {
            dim3 tb(32, 4, 1);
            dim3 gr((f.d.nx + 31) / 32, (f.d.ny + 3) / 4, f.d.nz);
            KT_BEGIN(K_MISC, g.stream);
            launch_pdl(k_mg_prolong_solution, gr, tb, g.stream, f.d, f.dev, c.d, c.dev, c.mg, f.nw);
            KT_END(K_MISC, g.stream);
        }
        {
            dim3 tb(32, 4, 2);
            dim3 gr((f.d.NI + 31) / 32, (f.d.NJ + 3) / 4, (f.d.NK + 1) / 2);
            KT_BEGIN(K_MISC, g.stream);
            launch_pdl(k_mg_extrapolate, gr, tb, g.stream, f.d, f.dev, f.nw);
            KT_END(K_MISC, g.stream);
        }
        const bool rans = g.prm.equations == ADFB_RANS;
        if (rans && launch_bc_levels(f.d, f.dev, f.subfaces, 1, 1, 0, g.stream)) return fail("turbulence BC launch failed");
        if (launch_bc_levels(f.d, f.dev, f.subfaces, 1, 0, 1, g.stream)) return fail("flow BC launch failed");
        if (launch_bc_levels(f.d, f.dev, f.subfaces, 1, 0, 1, g.stream)) return fail("flow BC launch failed");
    }
    int nwAll = 5;
    for (Block& f : g.blocks) if (f.alive && f.level == fineLevel) nwAll = f.nw;
    if (halo_exchange_impl(fineLevel, 1, nwAll, 1, 1, overset_present(fineLevel))) return 1;
    for (Block& f : g.blocks) {
        if (!f.alive || f.level != fineLevel) continue;
        if (launch_bc_levels(f.d, f.dev, f.subfaces, 1, 0, 1, g.stream)) return fail("flow BC launch failed");
    }
    if (halo_exchange_impl(fineLevel, 1, nwAll, 1, 1, overset_present(fineLevel))) return 1;
    CK(cudaGetLastError());
    return 0;
}
int adfb_mg_prolong_solution(int fineLevel) {
    ADFB_RANGE("adfb_mg_prolong_solution");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_mg_prolong_solution: adfb_set_params has not been called");
    if (fineLevel < 1 || g.groundLevel != fineLevel + 1)
        return fail("adfb_mg_prolong_solution: the ground level must be %d (adfb_set_ground_level), it is %d", fineLevel + 1, g.groundLevel);
    const unsigned long long key = (11ull << 40) | ((unsigned long long)fineLevel << 32);
    return run_graphed(key, [&]() { return adfb_mg_prolong_solution_body(fineLevel); });
}

// executeMGCycle, multiGrid.F90:825-955, for the cycling strategy of setCycleStrategy (:957-1030): entries
// -1 = prolongate to the next finer level, 0 = smoothing step, +1 = restrict to the next coarser level.
// Ground level 1.  The turbulence solve and the final residual of the cycle are included (:933-951).
static int adfb_mg_cycle_body(int nSteps, const int* cycling, int smoother) {
    const int ground = g.groundLevel;
    int level = ground;
    for (int n = 0; n < nSteps; n++) {
        switch (cycling[n]) {
            case -1:
                level -= 1;
                if (level < ground) return fail("adfb_mg_cycle: cycling strategy leaves the grid hierarchy");
                if (adfb_mg_prolong(level)) return 1;
                break;
            case 0:
                if (n > 0 && cycling[n - 1] != 1) {
                    if (adfb_timestep(level, 0)) return 1;
                    if (adfb_smoother_residual(level, 0)) return 1;
                }
                if (smoother == 0) { if (adfb_rk_cycle(level)) return 1; }
                else if (adfb_dadi_cycle(level, ground == 1 ? smoother : 1)) return 1;   // DADISmoother: nSubiterations steps on every level if groundLevel == 1, else one (smoothers.F90:400)
                break;
            case 1:
                if (adfb_mg_restrict(level)) return 1;
                level += 1;
                break;
            default: return fail("adfb_mg_cycle: cycling entry %d", cycling[n]);
        }
    }
    if (level != ground) return fail("adfb_mg_cycle: the strategy does not end on the ground level");
    if (g.prm.equations == ADFB_RANS)
        if (adfb_sa_ddadi(ground, g.prm.nSubiterTurb)) return 1;
    if (adfb_timestep(ground, 0)) return 1;
    return adfb_smoother_residual(ground, 0);
}
int adfb_mg_cycle(int nSteps, const int* cycling, int smoother) {
    ADFB_RANGE("adfb_mg_cycle");
    NEED_INIT();
    if (!g.havePrm) return fail("adfb_mg_cycle: adfb_set_params has not been called");
    if (nSteps < 1 || nSteps > 4096 || !cycling) return fail("adfb_mg_cycle: bad cycling strategy");
    if (smoother < 0 || smoother > 64) return fail("adfb_mg_cycle: smoother must be 0 (Runge-Kutta) or nSubiterations >= 1 (DADI)");
    unsigned long long h = 1469598103934665603ull;
    for (int n = 0; n < nSteps; n++) h = (h ^ (unsigned long long)(cycling[n] + 2)) * 1099511628211ull;
    h = (h ^ (unsigned long long)(smoother + 7)) * 1099511628211ull;
    const unsigned long long key = (10ull << 40) | (h & 0xffffffffffull);
    std::vector<int> cyc(cycling, cycling + nSteps);
    return run_graphed(key, [&]() { return adfb_mg_cycle_body(nSteps, cyc.data(), smoother); });
}

// ---------------------------------------------------------------------------
// Right-preconditioned restarted GMRES on the device for the matrix-free NK (op 0, adfb_mffd_set_base first) or ANK
// (op 1, adfb_ank_mffd_set_base first) operator: what PETSc's KSPGMRES does for NK_KSP / ANK_KSP
// (NKSolvers.F90:395-435, 2009-2037: GMRES, restart = subspace, right preconditioning, classical Gram-Schmidt without
// refinement, zero initial guess), with the Krylov vectors resident on the GPU.  The preconditioner (ASM/ILU of
// the assembled approximate Jacobian in the reference) stays outside: pc == NULL is the identity, otherwise
// pc(ctx, inDev, outDev, n) applies M^-1 to a device vector.
static int kry_apply_op(int op, const double* inDev, double* outDev, long long n) {
    if (op == 2) return ank_vec_kernel(inDev, nullptr, outDev, nullptr, 1.0, 4);   // y = timeStepMat x (linear)
    CK(cudaMemcpyAsync(g.nkA, inDev, n * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    const int rc = op == 0 ? mffd_core(n, -1.0) : ank_mffd_core(n, -1.0);
    if (rc == 1) return 1;
    if (rc == 2) CK(cudaMemsetAsync(outDev, 0, n * sizeof(double), g.stream));
    else CK(cudaMemcpyAsync(outDev, g.nkY, n * sizeof(double), cudaMemcpyDeviceToDevice, g.stream));
    return 0;
}
static int kry_dots(const double* V, long long ld, int nv, const double* w, long long n, double* hOut) {
    KT_BEGIN(K_MFFD, g.stream);
    k_multidot<<<ADFB_GMRES_PARTS, 256, 0, g.stream>>>(V, ld, nv, w, n, g.kryRed);
    KT_END(K_MFFD, g.stream);
    double* fin = g.kryRed + (size_t)ADFB_GMRES_PARTS * ADFB_GMRES_MAXV;
    KT_BEGIN(K_MFFD, g.stream);
    k_multidot_final<<<nv, 256, 0, g.stream>>>(g.kryRed, ADFB_GMRES_PARTS, nv, fin);
    KT_END(K_MFFD, g.stream);
    if (g.nranks > 1) {
        const int rc = g.nccl.AllReduce(fin, fin, nv, kNcclDouble, kNcclSum, g.comm, g.stream);
        if (rc != 0) return fail("ncclAllReduce: %s", g.nccl.GetErrorString(rc));
    }
    CK(cudaMemcpyAsync(g.hRed, fin, nv * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    for (int i = 0; i < nv; i++) hOut[i] = g.hRed[i];
    return 0;
}
int adfb_gmres_solve(int op, const double* rhs, double* x, long long n, int restart, int maxIts, double rtol, double atol,
                     AdfbPrecondFn pc, void* pcCtx, int* itsOut, double* resNormOut) {
    ADFB_RANGE("adfb_gmres_solve");
    NEED_INIT();
    if (!rhs || !x) return fail("adfb_gmres_solve: null vector");
    if (op < 0 || op > 2) return fail("adfb_gmres_solve: op must be 0 (NK product), 1 (ANK product) or 2 (time-step matrix)");
    if (restart < 1 || restart > ADFB_GMRES_MAXV - 2) return fail("adfb_gmres_solve: restart must be in 1..%d", ADFB_GMRES_MAXV - 2);
    if (maxIts < 1) return fail("adfb_gmres_solve: maxIts must be >= 1");
    long long need = 0;
    if (op == 0) {
        if (!g.nkHaveBase) return fail("adfb_gmres_solve: adfb_mffd_set_base has not been called");
        need = adfb_state_size();
    } else {
        if (ank_ready("adfb_gmres_solve", n, &need)) return 1;
        if (op == 1 && !g.ankHaveBase) return fail("adfb_gmres_solve: adfb_ank_mffd_set_base has not been called");
    }
    if (n != need) return fail("adfb_gmres_solve: vector length %lld != %lld", n, need);
    const int m = restart;
    const size_t nvec = (size_t)m + 4;   // V_0..V_m, w, z, xDev
    if (g.kryVN < nvec * (size_t)n) {
        if (g.kryV) cudaFree(g.kryV);
        g.kryV = nullptr; g.kryVN = 0;
        CK(cudaMalloc((void**)&g.kryV, nvec * (size_t)n * sizeof(double)));
        g.kryVN = nvec * (size_t)n;
    }
    if (!g.kryRed) CK(cudaMalloc((void**)&g.kryRed, ((size_t)ADFB_GMRES_PARTS + 1) * ADFB_GMRES_MAXV * sizeof(double)));
    if (!g.hRed) return fail("adfb_gmres_solve: reduction buffer missing");
    double* V = g.kryV;
    double* w = V + (size_t)(m + 1) * n;
    double* z = w + n;
    double* xd = z + n;
    const unsigned nb = (unsigned)((n + 255) / 256);
    CK(cudaMemsetAsync(xd, 0, n * sizeof(double), g.stream));
    // r0 = b (zero initial guess, like the reference's KSPs)
    CK(cudaMemcpyAsync(w, rhs, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
    double bb = 0.0;
    if (kry_dots(w, n, 1, w, n, &bb)) return 1;
    const double bnorm = sqrt(bb);
    double rnorm = bnorm;
    const double target = fmax(rtol * bnorm, atol);
    int its = 0;
    std::vector<double> H((size_t)(m + 1) * m), cs(m), sn(m), gg(m + 1), hcol(m + 2);
    bool first = true;
    while (its < maxIts && rnorm > target) {
        if (!first) {   // restart: r = b - A M^-1 ... with right preconditioning x already holds M^-1 (V y): r = b - A x
            if (kry_apply_op(op, xd, w, n)) return 1;
            CK(cudaMemcpyAsync(z, rhs, n * sizeof(double), cudaMemcpyHostToDevice, g.stream));
            GmresCoef c1 = {}; c1.c[0] = 1.0;
            k_axpy_many<<<nb, 256, 0, g.stream>>>(z, n, 1, c1, -1.0, w, n);   // w = -w + b
            if (kry_dots(w, n, 1, w, n, &bb)) return 1;
            rnorm = sqrt(bb);
            if (rnorm <= target) break;
        }
        first = false;
        k_scale_to<<<nb, 256, 0, g.stream>>>(w, 1.0 / rnorm, V, n);
        std::fill(gg.begin(), gg.end(), 0.0);
        gg[0] = rnorm;
        int j = 0;
        for (; j < m && its < maxIts; j++) {
            const double* vj = V + (size_t)j * n;
            const double* zin = vj;
            if (pc) {
                CK(cudaStreamSynchronize(g.stream));
                if (pc(pcCtx, vj, z, n)) return fail("adfb_gmres_solve: the preconditioner callback failed");
                zin = z;
            }
            if (kry_apply_op(op, zin, w, n)) return 1;
            // classical Gram-Schmidt: all projections from the unmodified w, then one update
            if (kry_dots(V, n, j + 1, w, n, hcol.data())) return 1;
            GmresCoef cf = {};
            for (int i = 0; i <= j; i++) cf.c[i] = -hcol[i];
            k_axpy_many<<<nb, 256, 0, g.stream>>>(V, n, j + 1, cf, 1.0, w, n);
            double ww = 0.0;
            if (kry_dots(w, n, 1, w, n, &ww)) return 1;
            hcol[j + 1] = sqrt(ww);
            if (hcol[j + 1] > 0.0) k_scale_to<<<nb, 256, 0, g.stream>>>(w, 1.0 / hcol[j + 1], V + (size_t)(j + 1) * n, n);
            // Givens rotations on the new column
            for (int i = 0; i < j; i++) {
                const double t = cs[i] * hcol[i] + sn[i] * hcol[i + 1];
                hcol[i + 1] = -sn[i] * hcol[i] + cs[i] * hcol[i + 1];
                hcol[i] = t;
            }
            const double den = hypot(hcol[j], hcol[j + 1]);
            cs[j] = den > 0.0 ? hcol[j] / den : 1.0;
            sn[j] = den > 0.0 ? hcol[j + 1] / den : 0.0;
            hcol[j] = den;
            gg[j + 1] = -sn[j] * gg[j];
            gg[j] = cs[j] * gg[j];
            for (int i = 0; i <= j; i++) H[(size_t)i + (size_t)(m + 1) * j] = hcol[i];
            its++;
            rnorm = fabs(gg[j + 1]);
            if (den == 0.0) break;   // exact breakdown with a zero column: solve with the first j columns only
            if (rnorm <= target) { j++; break; }
        }
        // y = H^-1 g (upper triangular), x += M^-1 (V y)
        const int k = j;
        std::vector<double> y(k);
        for (int i = k - 1; i >= 0; i--) {
            double t = gg[i];
            for (int l = i + 1; l < k; l++) t -= H[(size_t)i + (size_t)(m + 1) * l] * y[l];
            const double hii = H[(size_t)i + (size_t)(m + 1) * i];
            if (hii == 0.0) return fail("adfb_gmres_solve: singular Hessenberg matrix (breakdown at column %d)", i);
            y[i] = t / hii;
        }
        GmresCoef cy = {};
        for (int i = 0; i < k; i++) cy.c[i] = y[i];
        if (pc) {
            k_axpy_many<<<nb, 256, 0, g.stream>>>(V, n, k, cy, 0.0, w, n);
            CK(cudaStreamSynchronize(g.stream));
            if (pc(pcCtx, w, z, n)) return fail("adfb_gmres_solve: the preconditioner callback failed");
            GmresCoef c1 = {}; c1.c[0] = 1.0;
            k_axpy_many<<<nb, 256, 0, g.stream>>>(z, n, 1, c1, 1.0, xd, n);
        } else {
            k_axpy_many<<<nb, 256, 0, g.stream>>>(V, n, k, cy, 1.0, xd, n);
        }
    }
    CK(cudaMemcpyAsync(x, xd, n * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    CK(cudaGetLastError());
    if (itsOut) *itsOut = its;
    if (resNormOut) *resNormOut = rnorm;
    return 0;
}

int adfb_norms(double out[2]) {
    ADFB_RANGE("adfb_norms");
    NEED_INIT();
    if (!out) return fail("adfb_norms: null");
    out[0] = out[1] = 0.0;
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != 1) continue;
        const int nPart = 1024;
        if (g.dRedN < (size_t)2 * nPart + 2) {
            if (g.dRed) cudaFree(g.dRed);
            CK(cudaMalloc((void**)&g.dRed, (2 * nPart + 2) * sizeof(double)));
            g.dRedN = 2 * nPart + 2;
        }
        if (launch_norms(b.d, b.dev, b.nw, g.prm.turbResScale, g.dRed, nPart, g.stream)) return fail("norm kernel failed");
        CK(cudaMemcpyAsync(g.hRed, g.dRed + 2 * nPart, 2 * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
        CK(cudaStreamSynchronize(g.stream));
        out[0] += g.hRed[0];
        out[1] += g.hRed[1];
    }
    if (g.nranks > 1) {  // mpi_allreduce(monLoc, monGlob, ...), NKSolvers.F90:364
        g.hRed[0] = out[0]; g.hRed[1] = out[1];
        CK(cudaMemcpyAsync(g.dRed, g.hRed, 2 * sizeof(double), cudaMemcpyHostToDevice, g.stream));
        const int rc = g.nccl.AllReduce(g.dRed, g.dRed, 2, kNcclDouble, kNcclSum, g.comm, g.stream);
        if (rc != 0) return fail("ncclAllReduce: %s", g.nccl.GetErrorString(rc));
        CK(cudaMemcpyAsync(g.hRed, g.dRed, 2 * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
        CK(cudaStreamSynchronize(g.stream));
        out[0] = g.hRed[0]; out[1] = g.hRed[1];
    }
    return 0;
}

// getForces / wallIntegrationFace: Fp(3), Fv(3), Mp(3), Mv(3) over the wall subfaces of all local blocks of
// `level`, all-reduced.  The viscous part uses the wall stresses stored by the last adfb_residual call that had
// ADFB_RES_STORE_WALL set.
int adfb_forces(int level, const double refPoint[3], double pRef, double out[12]) {
    ADFB_RANGE("adfb_forces");
    NEED_INIT();
    if (!refPoint || !out) return fail("adfb_forces: null");
    if (g.dRedN < 16) {
        if (g.dRed) cudaFree(g.dRed);
        CK(cudaMalloc((void**)&g.dRed, 2050 * sizeof(double)));
        g.dRedN = 2050;
    }
    CK(cudaMemsetAsync(g.dRed, 0, 12 * sizeof(double), g.stream));
    for (Block& b : g.blocks) {
        if (!b.alive || b.level != level) continue;
        if (launch_wall_forces(b.d, b.dev, b.subfaces, refPoint, pRef, g.dRed, g.stream)) return fail("force kernel failed");
    }
    if (g.nranks > 1) {
        const int rc = g.nccl.AllReduce(g.dRed, g.dRed, 12, kNcclDouble, kNcclSum, g.comm, g.stream);
        if (rc != 0) return fail("ncclAllReduce: %s", g.nccl.GetErrorString(rc));
    }
    CK(cudaMemcpyAsync(g.hRed, g.dRed, 12 * sizeof(double), cudaMemcpyDeviceToHost, g.stream));
    CK(cudaStreamSynchronize(g.stream));
    for (int q = 0; q < 12; q++) out[q] = g.hRed[q];
    return 0;
}

}  // extern "C"
