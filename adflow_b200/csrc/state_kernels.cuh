// state_kernels.cuh -- cell-local state / geometry kernels
//
//   k_metrics    : face normals from node coordinates (blockette `metrics`,
//                  src/NKSolver/blockette.F90:854-960)
//   k_state_prep : computePressureSimple (src/utils/flowUtils.F90:867-930),
//                  computeLamViscosity (:1201-1323), saEddyViscosity
//                  (src/turbulence/turbUtils.F90:657-712) fused in one pass
//   k_norms      : sumResiduals / sumAllResiduals (src/utils/utils.F90:6364-6459), maxHdiffMach / maxEddyv
//                  (:2422-2531): the convergence monitor of adfb_monitor and adfb_norms
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
    ADFB_PDL_SYNC();  // launched with programmatic stream serialization (launch_kernel with pdl)
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

// The monitor values of convergenceInfo (solvers.F90:1338-1376) over the owned cells 2:il, 2:jl, 2:kl of one block, in
// the layout of adfb_monitor: 0..5 sumResiduals (utils.F90:6364-6398) of rho, rho u, rho v, rho w, rho E, nu~;
// 6 sumAllResiduals (:6400-6448); 7 max |(rhoE + p) / rho - hInf| and 8 max Mach^2 of maxHdiffMach (:2466-2531), before
// its division by hInf and square root; 9 max rev / rlv of maxEddyv (:2422-2464).
enum { ADFB_MON_N = 10, ADFB_MON_NSUM = 7 };
struct MonCoef {
    double turbResScale, hInf, gamma;
    int nw, eddy;   // eddy: an eddy-viscosity model (RANS), else maxEddyv is 0
};

// Two-pass deterministic reduction.  Pass 1, per block: CTA q of nPart writes its partial of value v to part[v nPart + q];
// a grid-stride loop of a fixed grid, then a fixed tree.  what: bit 0 the sums, bit 1 the maxima; a cleared bit skips
// the work and the loads behind it, and its partials are not written.  The maxima form each cell's value with explicit
// roundings (no FMA contraction), so they are the reference's bits; fmax ignores a NaN operand, so a NaN cell does not
// enter them.
__global__ void __launch_bounds__(256) k_norms_partial(Dims d, BlockDev b, MonCoef mc, unsigned what, double* part, int nPart) {
    __shared__ double s[ADFB_MON_N][256];
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    const bool sums = what & 1, maxima = what & 2;
    const int v0 = sums ? 0 : ADFB_MON_NSUM, v1 = maxima ? ADFB_MON_N : ADFB_MON_NSUM;
    double a[ADFB_MON_N];
#pragma unroll
    for (int v = 0; v < ADFB_MON_N; v++) a[v] = 0.0;
    const long long N = d.N;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < nOwned; q += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(q % d.nx) + 2;
        const int j = (int)((q / d.nx) % d.ny) + 2;
        const int k = (int)(q / ((long long)d.nx * d.ny)) + 2;
        const long long c = ADFB_IDX(i, j, k);
        if (sums) {
            const double vol = b.vol[c];
            const double ovv = 1.0 / vol;
            double ssum = 0.0;   // state_sum: the cell's terms in variable order, then added to the total
#pragma unroll
            for (int l = 0; l < 5; l++) {
                const double dw = b.dw[l * N + c];
                const double r = dw / vol;
                a[l] += r * r;
                const double t = dw * ovv;
                ssum += t * t;
            }
            for (int l = 5; l < mc.nw; l++) {
                const double dw = b.dw[l * N + c];
                const double r = dw / vol;
                a[5] += r * r;
                const double t = dw * ovv * mc.turbResScale;
                ssum += t * t;
            }
            a[6] += ssum;
        }
        if (maxima) {
            const double rho = b.w[c], u = b.w[N + c], v = b.w[2 * N + c], w = b.w[3 * N + c], p = b.p[c];
            const double hdiff = fabs(__dsub_rn(__ddiv_rn(__dadd_rn(b.w[4 * N + c], p), rho), mc.hInf));
            const double v2 = __dadd_rn(__dadd_rn(__dmul_rn(u, u), __dmul_rn(v, v)), __dmul_rn(w, w));
            const double mach2 = __ddiv_rn(__dmul_rn(v2, rho), __dmul_rn(mc.gamma, p));
            a[7] = fmax(a[7], hdiff);
            a[8] = fmax(a[8], mach2);
            if (mc.eddy) a[9] = fmax(a[9], __ddiv_rn(b.rev[c], b.rlv[c]));
        }
    }
#pragma unroll
    for (int v = 0; v < ADFB_MON_N; v++) s[v][threadIdx.x] = a[v];
    __syncthreads();
    for (int st = 128; st > 0; st >>= 1) {
        if ((int)threadIdx.x < st)
            for (int v = v0; v < v1; v++) {
                if (v < ADFB_MON_NSUM) s[v][threadIdx.x] += s[v][threadIdx.x + st];
                else s[v][threadIdx.x] = fmax(s[v][threadIdx.x], s[v][threadIdx.x + st]);
            }
        __syncthreads();
    }
    if ((int)threadIdx.x >= v0 && (int)threadIdx.x < v1) part[threadIdx.x * nPart + blockIdx.x] = s[threadIdx.x][0];
}

// Pass 2, one CTA: block bi's partials at part + bi stride reduced by a fixed tree, then the blocks combined in block
// order, sum = ((0 + b0) + b1) + ..., max from 0; out[7] / hInf and sqrt(out[8]) as maxHdiffMach ends (monotone, so
// they commute with the maximum over blocks and ranks).  Entries of a cleared `what` bit are 0.
__global__ void __launch_bounds__(256) k_norms_final(const double* __restrict__ part, int nPart, long long stride, int nBlk,
                                                     unsigned what, double hInf, double* __restrict__ out) {
    __shared__ double s[ADFB_MON_N][256];
    __shared__ double tot[ADFB_MON_N];
    if (threadIdx.x < ADFB_MON_N) tot[threadIdx.x] = 0.0;
    const int v0 = (what & 1) ? 0 : ADFB_MON_NSUM, v1 = (what & 2) ? ADFB_MON_N : ADFB_MON_NSUM;
    for (int bi = 0; bi < nBlk; bi++) {
        const double* pb = part + bi * stride;
        for (int v = v0; v < v1; v++) {
            double a = 0.0;
            if (v < ADFB_MON_NSUM) for (int q = threadIdx.x; q < nPart; q += 256) a += pb[v * nPart + q];
            else for (int q = threadIdx.x; q < nPart; q += 256) a = fmax(a, pb[v * nPart + q]);
            s[v][threadIdx.x] = a;
        }
        __syncthreads();
        for (int st = 128; st > 0; st >>= 1) {
            if ((int)threadIdx.x < st)
                for (int v = v0; v < v1; v++) {
                    if (v < ADFB_MON_NSUM) s[v][threadIdx.x] += s[v][threadIdx.x + st];
                    else s[v][threadIdx.x] = fmax(s[v][threadIdx.x], s[v][threadIdx.x + st]);
                }
            __syncthreads();
        }
        if (threadIdx.x == 0)
            for (int v = v0; v < v1; v++) tot[v] = v < ADFB_MON_NSUM ? tot[v] + s[v][0] : fmax(tot[v], s[v][0]);
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        if (what & 2) { tot[7] = __ddiv_rn(tot[7], hInf); tot[8] = __dsqrt_rn(tot[8]); }
        for (int v = 0; v < ADFB_MON_N; v++) out[v] = tot[v];
    }
}

// The per-call coefficients of the whole-state modes of k_vec, formed on the host: the free-stream change and the rotation
// of infChangeCorrection (modes 4, 5), the free-stream viscosities of setUniformFlow (mode 6)
struct VecCoef {
    double dWinf[5];     // wInf(1:5) - oldWinf
    double rot[9];       // rotMat(i, j) at [3 (i-1) + (j-1)] (getRotMatrix)
    double mag1, mag2;   // |old velocity|, |new velocity|
    double muInf, revInf;
};

// AoS <-> SoA vector kernels (getStates/setStates/getRes gather loops,
// src/NKSolver/NKSolvers.F90:1378-1485). mode 0: vec <- w ; 1: w <- vec ; 2: vec <- dw/volRef ;
// 3: w(0:ib, 0:jb, 0:kb, 1:nw) <- wInf, halos included (the uniform flow of getFreeStreamResidual, :298-312; vec unused).
// Whole-state modes (vec unused, coefficients in cf):
// 4: w(2:il, 2:jl, 2:kl, 1:5) += dWinf, one thread per owned cell ("offset" of infChangeCorrection,
//    src/initFlow/initializeFlow.F90:230-247)
// 5: owned velocity <- (rot v) * mag2 / mag1, rho and rhoE += their dWinf ("rotate", :249-284); explicit roundings, so that
//    no FMA contraction changes the reference's bits
// 6: setUniformFlow (:2143-2212) over the whole box, one thread per cell: w = wInf, dw = 0, fw = 0, p = pInfCorr,
//    rlv = muInf unless Euler, rev = eddyVisInfRatio * muInf for RANS
__global__ void __launch_bounds__(256) k_vec(Dims d, BlockDev b, int nw, double* vec, int mode, VecCoef cf) {
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    const long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (mode == 3) {
        if (q < d.N * nw) b.w[q] = c_prm.wInf[q / d.N];
        return;
    }
    if (mode == 6) {
        if (q >= d.N) return;
        for (int l = 0; l < nw; l++) { b.w[l * d.N + q] = c_prm.wInf[l]; b.dw[l * d.N + q] = 0.0; }
        for (int l = 0; l < 5; l++) b.fw[l * d.N + q] = 0.0;
        b.p[q] = c_prm.pInfCorr;
        if (c_prm.equations != ADFB_EULER) b.rlv[q] = cf.muInf;
        if (c_prm.equations == ADFB_RANS) b.rev[q] = cf.revInf;
        return;
    }
    if (mode >= 4) {
        if (q >= nOwned) return;
        const long long c = ADFB_IDX((int)(q % d.nx) + 2, (int)((q / d.nx) % d.ny) + 2, (int)(q / ((long long)d.nx * d.ny)) + 2);
        const long long N = d.N;
        if (mode == 4) {
            for (int l = 0; l < 5; l++) b.w[l * N + c] = __dadd_rn(b.w[l * N + c], cf.dWinf[l]);
            return;
        }
        const double v[3] = {b.w[N + c], b.w[2 * N + c], b.w[3 * N + c]};
        for (int m = 0; m < 3; m++) {
            // matmul(rotMat, vCell): ((r1 v1 + r2 v2) + r3 v3), then * mag2, then / mag1
            const double r = __dadd_rn(__dadd_rn(__dmul_rn(cf.rot[3 * m], v[0]), __dmul_rn(cf.rot[3 * m + 1], v[1])),
                                       __dmul_rn(cf.rot[3 * m + 2], v[2]));
            b.w[(m + 1) * N + c] = __ddiv_rn(__dmul_rn(r, cf.mag2), cf.mag1);
        }
        b.w[c] = __dadd_rn(b.w[c], cf.dWinf[0]);
        b.w[4 * N + c] = __dadd_rn(b.w[4 * N + c], cf.dWinf[4]);
        return;
    }
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

static int launch_vec(const Dims& d, const BlockDev& b, int nw, double* vec, int mode, cudaStream_t stream,
                      const VecCoef& cf = VecCoef()) {
    const long long nOwned = (long long)d.nx * d.ny * d.nz;
    // mode 3 covers the whole box per variable, 4 and 5 the owned cells, 6 the box cells
    const long long n = mode == 3 ? d.N * nw : mode == 6 ? d.N : mode >= 4 ? nOwned : nOwned * nw;
    launch_kernel(K_VEC, false, (unsigned)((n + 255) / 256), 256, 0, stream, k_vec, d, b, nw, vec, mode, cf);
    return (int)cudaGetLastError();
}

static int launch_metrics(const Dims& d, const BlockDev& b, int rightHanded, cudaStream_t stream) {
    dim3 tb(32, 4, 2);
    dim3 g((d.ie + 1 + tb.x - 1) / tb.x, (d.je + 1 + tb.y - 1) / tb.y, (d.ke + 1 + tb.z - 1) / tb.z);
    launch_kernel(K_METRICS, false, g, tb, 0, stream, k_metrics, d, b, rightHanded ? 0.5 : -0.5);
    return (int)cudaGetLastError();
}

static int launch_state_prep(const Dims& d, const BlockDev& b, const AdfbParams& prm, bool includeHalos, bool etot, cudaStream_t stream) {
    (void)prm;
    dim3 tb(32, 4, 2);
    const int ni = includeHalos ? d.NI : d.nx, nj = includeHalos ? d.NJ : d.ny, nk = includeHalos ? d.NK : d.nz;
    dim3 g((ni + tb.x - 1) / tb.x, (nj + tb.y - 1) / tb.y, (nk + tb.z - 1) / tb.z);
    launch_kernel(K_STATE, true, g, tb, 0, stream, k_state_prep, d, b, includeHalos ? 1 : 0, prm.equations == ADFB_RANS ? 6 : 5, etot ? 1 : 0, 0, INT_MAX);
    return (int)cudaGetLastError();
}

// pass 1 of the monitor reduction on one block, into its own nPart x ADFB_MON_N slot of the partials
static int launch_norms_partial(const Dims& d, const BlockDev& b, const MonCoef& mc, unsigned what, double* part, int nPart,
                                cudaStream_t stream) {
    launch_kernel(K_NORMS, false, nPart, 256, 0, stream, k_norms_partial, d, b, mc, what, part, nPart);
    return (int)cudaGetLastError();
}
static int launch_norms_final(const double* part, int nPart, long long stride, int nBlk, unsigned what, double hInf, double* out,
                              cudaStream_t stream) {
    launch_kernel(K_NORMS, false, 1, 256, 0, stream, k_norms_final, part, nPart, stride, nBlk, what, hInf, out);
    return (int)cudaGetLastError();
}
