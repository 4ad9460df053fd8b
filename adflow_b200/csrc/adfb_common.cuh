// adfb_common.cuh -- shared device-side definitions for libadflow_b200
//
// Data layout in HBM (DESIGN.md section 3): every per-block array lives in one
// uniform box (0:ib, 0:jb, 0:kb), i fastest, so the Fortran index (i,j,k) of the
// reference (src/modules/block.F90:205-752) is the device offset
// i + NI*(j + NJ*k) for cell, node and face arrays alike; multi-component
// arrays are SoA with the component slowest (w(i,j,k,l) -> l*N + idx), which is
// the reference's own ordering and gives unit-stride, fully coalesced access
// along i for every variable.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <nvtx3/nvToolsExt.h>   // header-only; ranges are no-ops unless a profiler is attached
#include "../../include/adflow_b200.h"

struct Dims {
    int nx, ny, nz;
    int il, jl, kl, ie, je, ke, ib, jb, kb;
    int NI, NJ, NK;
    long long N;   // box size
    long long sJ, sK;  // strides (sI == 1)
};

static inline Dims make_dims(int nx, int ny, int nz) {
    Dims d;
    d.nx = nx; d.ny = ny; d.nz = nz;
    d.il = nx + 1; d.jl = ny + 1; d.kl = nz + 1;
    d.ie = nx + 2; d.je = ny + 2; d.ke = nz + 2;
    d.ib = nx + 3; d.jb = ny + 3; d.kb = nz + 3;
    d.NI = d.ib + 1; d.NJ = d.jb + 1; d.NK = d.kb + 1;
    d.N = (long long)d.NI * d.NJ * d.NK;
    d.sJ = d.NI; d.sK = (long long)d.NI * d.NJ;
    return d;
}

// device pointers of one block (all in the uniform box)
struct BlockDev {
    double *w, *p, *rlv, *rev;          // state
    double *x, *si, *sj, *sk;           // geometry (3 comps each)
    double *vol, *volRef, *d2Wall;
    int8_t *porI, *porJ, *porK;
    int32_t *iblank;
    double *dw, *fw;                    // residual (nw) and dissipative+viscous part (5)
    double *ss, *dss;                   // entropy / shock sensor (3)
    double *aa, *radI, *radJ, *radK, *dtl;
    double *grad;                       // 12 nodal gradient arrays
    double *wn, *pn;                    // RK stage-0 copies (5 / 1)
    double *scratch;                    // 10 work arrays (DADI, SA solve)
    // geometry-derived static arrays (k_geom) and the face-flux store
    double *ssum;                       // 9: s(c-sd)+s(c) per direction
    double *sv;                         // 9: dual-face normal sums per direction
    double *ovol;                       // 1: 1/(8-cell volume sum) at nodes
    double *vn;                         // 12: cell-centre unit vector + 1/length per face direction
    double *flux;                       // 30: face fluxes (15 used in merged mode)
    double *shock;                      // frozen shock sensor (referenceShockSensor)
    // viscSubface%tau / %q of the six block-boundary face planes (storeWallTensor): [dir][side][9][plane], plane
    // stride wallP, in-plane index ia + (dir == 0 ? NJ : NI) * jb
    double *wallTau;
    long long wallP;
    // multigrid: residual forcing term (5), solution at the start of the coarse-level visit (5 / 1), and the
    // level flag: coarse = 1 on levels > 1 (no directional scaling of the radii, constant-pressure walls, frozen
    // eddy viscosity, first-order dissipation: the currentLevel > groundLevel branches of the reference)
    double *wr, *w1, *p1;
    int coarse;
};

// Matrix-free product fused into the residual (NKSolvers.F90:437-461 with setW :1331 and setRVec :1262): the kernels that
// write dw also form y = (dw / volRef [* turbResScale] - F0) / h of their rows.  The record lives in device memory (one per
// context) and is rewritten before every product, so the captured graph of the residual keeps working with a new h.
struct MffdDev {
    const double* F0;   // base residual F(U), AoS per owned cell like getStates
    double* y;          // result
    double h;
    int nw;
};
struct MffdEpi {        // per block: the record + offset of the block's first owned cell in the vectors
    const MffdDev* rec; // nullptr: no fused epilogue
    long long cell0;
};
__host__ __device__ inline void mffd_epilogue(const MffdEpi& m, const Dims& d, int i, int j, int k, int l, double dwv, double volRef, double turbScale) {
    const MffdDev& R = *m.rec;
    const long long q = (m.cell0 + ((long long)(k - 2) * d.ny + (j - 2)) * d.nx + (i - 2)) * R.nw + l;
    const double ovv = 1.0 / volRef;
#if defined(__CUDA_ARCH__)
    // every step rounded on its own (no contraction), exactly as k_nkvec forms setRVec and the difference quotient
    double r = __dmul_rn(dwv, ovv);
    if (l >= 5) r = __dmul_rn(r, turbScale);
    R.y[q] = __ddiv_rn(__dsub_rn(r, R.F0[q]), R.h);
#else
    double r = dwv * ovv;
    if (l >= 5) r = r * turbScale;
    R.y[q] = (r - R.F0[q]) / R.h;
#endif
}

// single translation unit (adflow_b200.cu includes every *_kernels.cuh)
__constant__ AdfbParams c_prm;
// parameter-only constants of the flux kernels: [0], [1] the heat-flux coefficients 1/(Pr (gamma-1)), 1/(Pr_t (gamma-1)) of
// viscousFlux (formed on the host), [2] the shock-sensor floor sslim = 0.001 pInfCorr / rhoInf**gamma (blockette.F90:3060-3070;
// formed ON THE DEVICE by k_param_consts, so that it is bit for bit the value the kernels used to recompute with pow() per
// face and thread -- one 190-instruction pow chain per face otherwise: 21 % of the tile kernel's instructions)
// [3] = 1/rsaCb3, [4] = 1/rsaK**2 of the SA model, [7] = 1/(gamma-1), [8] = 1e-6 gamma pInfCorr / rhoInf (host quotients: correctly
// rounded on both sides); [5] = rhoInf**gamma / pInfCorr, [6] = sqrt(gamma pInfCorr / rhoInf) of the far-field BC (device)
__constant__ double c_fheat[16];
// Programmatic dependent launch: every PDL-launched kernel first waits for its predecessor (grid dependency sync: the
// predecessor has completed and its writes are visible), then -- with ADFB_PDL_TRIGGER=1 -- signals at once that ITS
// dependent may be launched, so that the dependent's blocks are scheduled while this kernel's last wave drains; the
// dependent still waits at its own grid dependency sync before touching memory.
__constant__ int c_pdlTrigger;
#define ADFB_PDL_SYNC()                                                  \
    do {                                                                 \
        cudaGridDependencySynchronize();                                 \
        if (c_pdlTrigger) cudaTriggerProgrammaticLaunchCompletion();     \
    } while (0)

#define ADFB_IDX(i, j, k) ((long long)(i) + d.sJ * (long long)(j) + d.sK * (long long)(k))

__host__ __device__ static inline double dmax_(double a, double b) { return a > b ? a : b; }
__host__ __device__ static inline double dmin_(double a, double b) { return a < b ? a : b; }

// ---------------------------------------------------------------------------
// launch accounting + optional per-kernel CUDA-event timing (bench.py roofline)
#include <vector>
enum KernelId { K_PREP = 0, K_NODAL, K_RESID, K_DIV, K_SA, K_STATE, K_METRICS, K_NORMS, K_VEC, K_BC, K_RK, K_HALO, K_DADI, K_SASOLVE, K_MFFD, K_MISC, K_NUM };
static const char* const kKernelNames[K_NUM] = {"k_prep", "k_nodal", "k_flowres|k_faces", "k_div", "k_sa", "k_state_prep", "k_metrics", "k_norms",
                                                "k_vec", "k_bc", "k_rk", "k_halo", "k_dadi", "k_sa_solve", "k_mffd", "k_misc"};
struct KTimer {
    bool on = false;
    long long launches = 0;
    long long count[K_NUM] = {0};
    double ms[K_NUM] = {0};
    struct Rec { int id; cudaEvent_t a, b; };
    std::vector<Rec> pending;
    std::vector<cudaEvent_t> pool;
    cudaEvent_t get() {
        if (!pool.empty()) { cudaEvent_t e = pool.back(); pool.pop_back(); return e; }
        cudaEvent_t e; cudaEventCreate(&e); return e;
    }
    void begin(int id, cudaStream_t s) {
        if (!on) return;
        Rec r; r.id = id; r.a = get(); r.b = get();
        cudaEventRecord(r.a, s);
        pending.push_back(r);
    }
    void end(int id, cudaStream_t s) {
        launches++; count[id]++;
        if (!on) return;
        cudaEventRecord(pending.back().b, s);
    }
    void collect() {  // caller has synchronised the stream
        for (Rec& r : pending) {
            float t = 0.f;
            cudaEventElapsedTime(&t, r.a, r.b);
            ms[r.id] += t;
            pool.push_back(r.a); pool.push_back(r.b);
        }
        pending.clear();
    }
    void reset() { collect(); for (int i = 0; i < K_NUM; i++) { ms[i] = 0; count[i] = 0; } }
};
static KTimer g_kt;

// What the launch helpers need of the context: properties of the device it is bound to and the side stream of the SA row.
// adfb_init reads and creates them for the device it binds, adfb_finalize releases them.
struct LaunchEnv {
    int nSM = 0;                 // multiprocessors
    size_t smemOptin = 0;        // opt-in dynamic shared memory per CTA
    // the SA row of the residual runs here beside the flow rows (launch_residual_core)
    cudaStream_t saStream = nullptr;
    cudaEvent_t saFork = nullptr, saJoin = nullptr;
};

// lanes per line for the partitioned Thomas kernels (tridiag_part.cuh): 8 lanes x <= 16 rows, 16 lanes x <= 16
// rows, or 0 = one thread per line (short or very long lines).
static inline int adfb_part_lanes(int nl) {
    if (nl >= 16 && nl <= 128) return 8;
    if (nl > 128 && nl <= 256) return 16;
    return 0;
}
// every launch site sits in an NVTX range named after its kernel family (SURVEY section 5: tracing)
#define KT_BEGIN(id, stream) do { nvtxRangePushA(kKernelNames[id]); g_kt.begin(id, stream); } while (0)
#define KT_END(id, stream) do { g_kt.end(id, stream); nvtxRangePop(); } while (0)
struct AdfbRange {   // NVTX range of one C-ABI entry point
    explicit AdfbRange(const char* name) { nvtxRangePushA(name); }
    ~AdfbRange() { nvtxRangePop(); }
};
#define ADFB_RANGE(name) AdfbRange adfb_range_(name)

// ---------------------------------------------------------------------------
// Launch with the programmatic-dependent-launch attribute (the kernel must call
// cudaGridDependencySynchronize() before touching memory).  ADFB_PDL=0 falls back to a plain launch.
template <typename... KArgs, typename... Args>
static void launch_pdl(void (*kern)(KArgs...), dim3 g, dim3 tb, cudaStream_t s, Args... args) {
    static int pdl = -1;
    if (pdl < 0) { const char* e = getenv("ADFB_PDL"); pdl = e ? atoi(e) : 1; }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = g; cfg.blockDim = tb; cfg.dynamicSmemBytes = 0; cfg.stream = s;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
    cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}

