// state_kernels.cuh -- cell-local state / geometry kernels
//
//   k_metrics    : face normals from node coordinates (blockette `metrics`,
//                  src/NKSolver/blockette.F90:854-960)
//   k_state_prep : computePressureSimple (src/utils/flowUtils.F90:867-930),
//                  computeLamViscosity (:1201-1323), saEddyViscosity
//                  (src/turbulence/turbUtils.F90:657-712) fused in one pass
//   k_norms      : sumResiduals / sumAllResiduals (src/utils/utils.F90:6364-6459)
#pragma once
#include <limits.h>
#include "adfb_common.cuh"
#include <math.h>

namespace {

__global__ void __launch_bounds__(256) k_metrics(Dims d, BlockDev b, double fact) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int j = blockIdx.y * blockDim.y + threadIdx.y;
    const int k = blockIdx.z * blockDim.z + threadIdx.z;
    if (i > d.ie || j > d.je || k > d.ke) return;
    const long long N = d.N;
    const long long c = ADFB_IDX(i, j, k);
    const double* x = b.x;
    double v1[3], v2[3];
    // i-face: i=0..ie, j=1..je, k=1..ke
    if (j >= 1 && k >= 1) {
        const long long jn = c - d.sK, mk = c - d.sJ, mn = c - d.sJ - d.sK;
#pragma unroll
        for (int m = 0; m < 3; m++) { v1[m] = x[m * N + jn] - x[m * N + mk]; v2[m] = x[m * N + c] - x[m * N + mn]; }
        b.si[c] = fact * (v1[1] * v2[2] - v1[2] * v2[1]);
        b.si[N + c] = fact * (v1[2] * v2[0] - v1[0] * v2[2]);
        b.si[2 * N + c] = fact * (v1[0] * v2[1] - v1[1] * v2[0]);
    }
    // j-face: i=1..ie, j=0..je, k=1..ke
    if (i >= 1 && k >= 1) {
        const long long ijn = c - d.sK, ljk = c - 1, ljn = c - 1 - d.sK;
#pragma unroll
        for (int m = 0; m < 3; m++) { v1[m] = x[m * N + ijn] - x[m * N + ljk]; v2[m] = x[m * N + ljn] - x[m * N + c]; }
        b.sj[c] = fact * (v1[1] * v2[2] - v1[2] * v2[1]);
        b.sj[N + c] = fact * (v1[2] * v2[0] - v1[0] * v2[2]);
        b.sj[2 * N + c] = fact * (v1[0] * v2[1] - v1[1] * v2[0]);
    }
    // k-face: i=1..ie, j=1..je, k=0..ke
    if (i >= 1 && j >= 1) {
        const long long lmk = c - 1 - d.sJ, ljk = c - 1, imk = c - d.sJ;
#pragma unroll
        for (int m = 0; m < 3; m++) { v1[m] = x[m * N + c] - x[m * N + lmk]; v2[m] = x[m * N + ljk] - x[m * N + imk]; }
        b.sk[c] = fact * (v1[1] * v2[2] - v1[2] * v2[1]);
        b.sk[N + c] = fact * (v1[2] * v2[0] - v1[0] * v2[2]);
        b.sk[2 * N + c] = fact * (v1[0] * v2[1] - v1[1] * v2[0]);
    }
}

// p on [pLo,pHi] (owned, or 0:ib with halos), rlv/rev on [vLo,vHi] (owned, or 1:ie with halos)
// kOff / kTop: the planes lo + kOff .. kTop only (slab pipeline of adfb_form_function); 0 / INT_MAX: all of them
__global__ void __launch_bounds__(256) k_state_prep(Dims d, BlockDev b, int includeHalos, int nw, int etot, int kOff, int kTop) {
    ADFB_PDL_SYNC();  // launched with programmatic stream serialization (launch_pdl)
    const int lo = includeHalos ? 0 : 2;
    const int i = blockIdx.x * blockDim.x + threadIdx.x + lo;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + lo;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + lo + kOff;
    const int iHi = includeHalos ? d.ib : d.il, jHi = includeHalos ? d.jb : d.jl, kHi = includeHalos ? d.kb : d.kl;
    if (i > iHi || j > jHi || k > kHi || k > kTop) return;
    const long long N = d.N;
    const long long c = ADFB_IDX(i, j, k);
    const double rho = b.w[c], u = b.w[N + c], v = b.w[2 * N + c], w = b.w[3 * N + c];
    const double v2 = u * u + v * v + w * w;
    double p = (c_prm.gammaInf - 1.0) * (b.w[4 * N + c] - 0.5 * rho * v2);
    p = dmax_(p, 1.e-4 * c_prm.pInfCorr);
    b.p[c] = p;
    // whalo2's computeEtotBlock on owned cells (haloExchange.F90:174-197), fused here
    if (etot) b.w[4 * N + c] = c_fheat[7] /* 1/(gamma-1) */ * p + 0.5 * rho * v2;
    if (c_prm.equations == ADFB_EULER) return;
    if (includeHalos && (i < 1 || i > d.ie || j < 1 || j > d.je || k < 1 || k > d.ke)) return;
    const double T = p / (c_prm.RGas * rho);
    const double rlv = c_prm.muSuth * ((c_prm.TSuth + c_prm.SSuth) / (T + c_prm.SSuth)) * pow(T / c_prm.TSuth, 1.5);
    b.rlv[c] = rlv;
    if (c_prm.equations != ADFB_RANS || nw < 6 || b.coarse) return;  // computeEddyViscosity: ground level only
    const double rnuSA = b.w[5 * N + c] * rho;
    const double chi = rnuSA / rlv;
    const double chi3 = chi * chi * chi;
    const double cv13 = c_prm.rsaCv1 * c_prm.rsaCv1 * c_prm.rsaCv1;
    b.rev[c] = chi3 / (chi3 + cv13) * rnuSA;
}

// referenceShockSensor (src/adjoint/adjointUtils.F90:1900-1950); disc: the discretisation of the residual that reads it
__global__ void __launch_bounds__(256) k_shock(Dims d, BlockDev b, int disc) {
    const long long c = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= d.N) return;
    const double p = b.p[c];
    // pressure for Euler and for matrix dissipation, entropy otherwise (adjointUtils.F90:1930-1947)
    b.shock[c] = (c_prm.equations == ADFB_EULER || disc == ADFB_DISS_MATRIX) ? p : p / pow(b.w[c], c_prm.gammaInf);
}

// computeEtotBlock(2,il,2,jl,2,kl) (src/utils/flowUtils.F90:551-672, cpConstant)
__global__ void __launch_bounds__(256) k_etot_owned(Dims d, BlockDev b) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const long long N = d.N, c = ADFB_IDX(i, j, k);
    const double r = b.w[c], u = b.w[N + c], v = b.w[2 * N + c], w = b.w[3 * N + c];
    b.w[4 * N + c] = c_fheat[7] /* 1/(gamma-1) */ * b.p[c] + 0.5 * r * (u * u + v * v + w * w);
}

// two-pass deterministic reduction: pass 1 -> nPart partial pairs, pass 2 -> final pair
__global__ void __launch_bounds__(256) k_norms_partial(Dims d, BlockDev b, int nw, double turbResScale, double* part, int nPart) {
    __shared__ double s0[256], s1[256];
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    double a0 = 0.0, a1 = 0.0;
    const long long N = d.N;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nOwned; q += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(q % d.nx) + 2;
        const int j = (int)((q / d.nx) % d.ny) + 2;
        const int k = (int)(q / ((long long)d.nx * d.ny)) + 2;
        const long long c = ADFB_IDX(i, j, k);
        const double ovv = 1.0 / b.vol[c];
        const double r = b.dw[c] / b.vol[c];
        a0 += r * r;
        double ssum = 0.0;
        for (int l = 0; l < 5; l++) { const double t = b.dw[l * N + c] * ovv; ssum += t * t; }
        for (int l = 5; l < nw; l++) { const double t = b.dw[l * N + c] * ovv * turbResScale; ssum += t * t; }
        a1 += ssum;
    }
    s0[threadIdx.x] = a0; s1[threadIdx.x] = a1;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if ((int)threadIdx.x < st) { s0[threadIdx.x] += s0[threadIdx.x + st]; s1[threadIdx.x] += s1[threadIdx.x + st]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { part[blockIdx.x] = s0[0]; part[nPart + blockIdx.x] = s1[0]; }
}
__global__ void __launch_bounds__(256) k_norms_final(double* part, int nPart) {
    __shared__ double s0[256], s1[256];
    double a0 = 0.0, a1 = 0.0;
    for (int q = threadIdx.x; q < nPart; q += 256) { a0 += part[q]; a1 += part[nPart + q]; }
    s0[threadIdx.x] = a0; s1[threadIdx.x] = a1;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if ((int)threadIdx.x < st) { s0[threadIdx.x] += s0[threadIdx.x + st]; s1[threadIdx.x] += s1[threadIdx.x + st]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { part[2 * nPart] = s0[0]; part[2 * nPart + 1] = s1[0]; }
}

// AoS <-> SoA vector kernels (getStates/setStates/getRes gather loops,
// src/NKSolver/NKSolvers.F90:1378-1485). mode 0: vec <- w ; 1: w <- vec ; 2: vec <- dw/volRef
__global__ void __launch_bounds__(256) k_vec(Dims d, BlockDev b, int nw, double* vec, int mode) {
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nOwned * nw) return;
    const int l = (int)(q % nw);
    const long long cell = q / nw;
    const int i = (int)(cell % d.nx) + 2;
    const int j = (int)((cell / d.nx) % d.ny) + 2;
    const int k = (int)(cell / ((long long)d.nx * d.ny)) + 2;
    const long long c = ADFB_IDX(i, j, k);
    if (mode == 0) vec[q] = b.w[l * d.N + c];
    else if (mode == 1) b.w[l * d.N + c] = vec[q];
    else vec[q] = b.dw[l * d.N + c] * (1.0 / b.volRef[c]);
}

// NK / MFFD vector kernels (src/NKSolver/NKSolvers.F90):
//  mode 0: setW (:1331-1376)            w <- vec, turbulence clipped at 1e-6*wInf
//  mode 1: perturbed setW               w <- max-clip(base + h*vec)   (MFFD: F(U + h a))
//  mode 2: setRVec (:1262-1329)         out <- dw/volRef (* turbResScale on turbulence rows)
//  mode 3: MFFD difference              out <- (dw/volRef*scale - base) / h
// q0 / qEnd: the entries q0 .. qEnd-1 of the block's vector only (slab pipeline); 0 / LLONG_MAX: all
__global__ void __launch_bounds__(256) k_nkvec(Dims d, BlockDev b, int nw, const double* __restrict__ vec,
                                               const double* __restrict__ base, double* __restrict__ out, double h, int mode, long long q0,
                                               long long qEnd) {
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    const long long q = q0 + (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nOwned * nw || q >= qEnd) return;
    const int l = (int)(q % nw);
    const long long cell = q / nw;
    const int i = (int)(cell % d.nx) + 2;
    const int j = (int)((cell / d.nx) % d.ny) + 2;
    const int k = (int)(cell / ((long long)d.nx * d.ny)) + 2;
    const long long c = ADFB_IDX(i, j, k);
    if (mode <= 1) {
        // U + h a as PETSc's VecWAXPY forms it (product rounded, then the sum: no contraction), identically in k_nkvec_prep
        double v = mode == 0 ? vec[q] : __dadd_rn(base[q], __dmul_rn(h, vec[q]));
        if (l >= 5) v = dmax_(1e-6 * c_prm.wInf[l], v);
        b.w[l * d.N + c] = v;
    } else {
        const double ovv = 1.0 / b.volRef[c];
        double r = __dmul_rn(b.dw[l * d.N + c], ovv);   // setRVec; each step rounded on its own, like mffd_epilogue
        if (l >= 5) r = __dmul_rn(r, c_prm.turbResScale);
        out[q] = mode == 2 ? r : __ddiv_rn(__dsub_rn(r, base[q]), h);
    }
}

// sum of squares of a device vector (two-pass, deterministic): part[0..nPart) then part[nPart]
// setW(U + h a) fused with the cell-local preamble of blocketteRes: one pass over the owned cells forms the perturbed state
// (turbulence clip of setW, NKSolvers.F90:1331-1376) and from it p, rhoE, rlv, rev exactly as k_state_prep does
__global__ void __launch_bounds__(256) k_nkvec_prep(Dims d, BlockDev b, int nw, const double* __restrict__ vec, const double* __restrict__ base,
                                                    const MffdDev* __restrict__ rec, int etot) {
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    const long long cell = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (cell >= nOwned) return;
    const int i = (int)(cell % d.nx) + 2, j = (int)((cell / d.nx) % d.ny) + 2, k = (int)(cell / ((long long)d.nx * d.ny)) + 2;
    const long long N = d.N, c = ADFB_IDX(i, j, k);
    const double h = rec->h;
    double wv[6];
    for (int l = 0; l < nw; l++) {
        const long long q = cell * nw + l;
        double v = __dadd_rn(base[q], __dmul_rn(h, vec[q]));
        if (l >= 5) v = dmax_(1e-6 * c_prm.wInf[l], v);
        wv[l] = v;
        b.w[l * N + c] = v;
    }
    const double rho = wv[0], u = wv[1], v = wv[2], w = wv[3];
    const double v2 = u * u + v * v + w * w;
    double p = (c_prm.gammaInf - 1.0) * (wv[4] - 0.5 * rho * v2);
    p = dmax_(p, 1.e-4 * c_prm.pInfCorr);
    b.p[c] = p;
    if (etot) b.w[4 * N + c] = c_fheat[7] /* 1/(gamma-1) */ * p + 0.5 * rho * v2;
    if (c_prm.equations == ADFB_EULER) return;
    const double T = p / (c_prm.RGas * rho);
    const double rlv = c_prm.muSuth * ((c_prm.TSuth + c_prm.SSuth) / (T + c_prm.SSuth)) * pow(T / c_prm.TSuth, 1.5);
    b.rlv[c] = rlv;
    if (c_prm.equations != ADFB_RANS || nw < 6 || b.coarse) return;
    const double rnuSA = wv[5] * rho;
    const double chi = rnuSA / rlv;
    const double chi3 = chi * chi * chi;
    const double cv13 = c_prm.rsaCv1 * c_prm.rsaCv1 * c_prm.rsaCv1;
    b.rev[c] = chi3 / (chi3 + cv13) * rnuSA;
}

__global__ void __launch_bounds__(256) k_sumsq_partial(const double* __restrict__ v, long long n, double* part) {
    __shared__ double s[256];
    double a = 0.0;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x) a += v[q] * v[q];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if ((int)threadIdx.x < st) s[threadIdx.x] += s[threadIdx.x + st];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[blockIdx.x] = s[0];
}
__global__ void __launch_bounds__(256) k_sum_final(double* part, int nPart) {
    __shared__ double s[256];
    double a = 0.0;
    for (int q = threadIdx.x; q < nPart; q += 256) a += part[q];
    s[threadIdx.x] = a;
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if ((int)threadIdx.x < st) s[threadIdx.x] += s[threadIdx.x + st];
        __syncthreads();
    }
    if (threadIdx.x == 0) part[nPart] = s[0];
}

}  // namespace

static int launch_vec(const Dims& d, const BlockDev& b, int nw, double* vec, int mode, cudaStream_t stream) {
    const long long n = (long long)d.nx * d.ny * d.nz * nw;
    KT_BEGIN(K_VEC, stream);
    k_vec<<<(unsigned)((n + 255) / 256), 256, 0, stream>>>(d, b, nw, vec, mode);
    KT_END(K_VEC, stream);
    return (int)cudaGetLastError();
}

static int launch_metrics(const Dims& d, const BlockDev& b, int rightHanded, cudaStream_t stream) {
    dim3 tb(32, 4, 2);
    dim3 g((d.ie + 1 + tb.x - 1) / tb.x, (d.je + 1 + tb.y - 1) / tb.y, (d.ke + 1 + tb.z - 1) / tb.z);
    KT_BEGIN(K_METRICS, stream);
    k_metrics<<<g, tb, 0, stream>>>(d, b, rightHanded ? 0.5 : -0.5);
    KT_END(K_METRICS, stream);
    return (int)cudaGetLastError();
}

static int launch_state_prep(const Dims& d, const BlockDev& b, const AdfbParams& prm, bool includeHalos, bool etot, cudaStream_t stream) {
    (void)prm;
    dim3 tb(32, 4, 2);
    const int ni = includeHalos ? d.NI : d.nx, nj = includeHalos ? d.NJ : d.ny, nk = includeHalos ? d.NK : d.nz;
    dim3 g((ni + tb.x - 1) / tb.x, (nj + tb.y - 1) / tb.y, (nk + tb.z - 1) / tb.z);
    KT_BEGIN(K_STATE, stream);
    launch_pdl(k_state_prep, g, tb, stream, d, b, includeHalos ? 1 : 0, prm.equations == ADFB_RANS ? 6 : 5, etot ? 1 : 0, 0, INT_MAX);
    KT_END(K_STATE, stream);
    return (int)cudaGetLastError();
}

static int launch_norms(const Dims& d, const BlockDev& b, int nw, double turbResScale, double* part, int nPart,
                        cudaStream_t stream) {
    KT_BEGIN(K_NORMS, stream);
    k_norms_partial<<<nPart, 256, 0, stream>>>(d, b, nw, turbResScale, part, nPart);
    KT_END(K_NORMS, stream);
    KT_BEGIN(K_NORMS, stream);
    k_norms_final<<<1, 256, 0, stream>>>(part, nPart);
    KT_END(K_NORMS, stream);
    return (int)cudaGetLastError();
}
