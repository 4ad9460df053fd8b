// dadi_kernels.cuh -- diagonalised ADI smoother (computedwDADI, src/solver/residuals.F90:1062-1748;
// executeDADIStep, src/solver/smoothers.F90:425-693)
//
// The reference makes 3 sweeps (j, i, k); each solves, for every grid line, 5 scalar
// tridiagonal systems (3 distinct coefficient sets: u+-0, u+c, u-c) with the Thomas
// algorithm (tridiagsolve, :1750-1783), and wraps the sweeps in cell-local changes of
// basis (T_eta^-1 :1277-1327, T_xi^-1 T_eta :1407-1448, T_zeta^-1 T_xi :1543-1583,
// T_zeta :1679-1731).  Each sweep is k_dadi_coef (cell coefficients, incoming change of
// basis), k_dadi_tri (tridiagonal rows) and a Thomas walk; after the k sweep k_dadi_post
// applies T_zeta and the -1/vol scaling (layout of the work arrays above k_dadi_coef).
// j and k lines are walked by k_dadi_thomas, one thread per (line, variable), threads
// adjacent in i (coalesced); i lines by k_dadi_thomas_tile, one warp per 32 lines.
//
// Reference quirks kept: the spectral_* terms are multiplied by zero (:1269-1271) and
// vanish; the k sweep's eps2 metric uses sj for the lower face (:1625-1627).
#pragma once
#include "adfb_common.cuh"
#include <math.h>

namespace {

struct DadiCoef {      // per cell, per direction
    double dP[3], dM[3];   // diagPlus / diagMinus for (u), (u+c), (u-c)
    double vt1, vt3;       // viscTerm1, viscTerm3
    double dtrb;           // dual_dt * max(iblank,0)
};

// cell-local coefficients of cell c for the sweep along sd (residuals.F90:1345-1372 etc.)
__device__ __forceinline__ void dadi_cell(const BlockDev& b, int N, int c, int sd, const double* __restrict__ s,
                                          const double* __restrict__ slow, double cfl, bool viscous, bool eddy, DadiCoef& A) {
    const double epsval = 0.08, fac = 1.05;
    const double cInf2 = c_prm.gammaInf * c_prm.pInf / c_prm.rhoInf;
    const double rho = b.w[c], vol = b.vol[c];
    const double volhalf = 0.5 / vol;
    // metterm(m) (face c|c+sd) and metterm(m-1) (face c-sd|c)
    double mp = 0.0, mm = 0.0;
    {
        double mut = 0.0;
        if (viscous) mut = b.rlv[c] + b.rlv[c + sd];
        if (eddy) mut = mut + b.rev[c] + b.rev[c + sd];
        const double volfact = 1.0 / (vol + b.vol[c + sd]);
        const double mt = s[c] * s[c] + s[N + c] * s[N + c] + s[2 * N + c] * s[2 * N + c];
        mp = mt * mut * volfact;
        const int cm = c - sd;
        mut = 0.0;
        if (viscous) mut = b.rlv[cm] + b.rlv[c];
        if (eddy) mut = mut + b.rev[cm] + b.rev[c];
        const double volfactm = 1.0 / (b.vol[cm] + vol);
        const double mtm = s[cm] * s[cm] + s[N + cm] * s[N + cm] + s[2 * N + cm] * s[2 * N + cm];
        mm = mtm * mut * volfactm;
    }
    A.vt1 = mp / vol / rho;
    A.vt3 = mm / vol / rho;
    // qq, cc (:1169-1211) use the true face sum; eps2 uses (s[c] + slow[c-sd]) (quirk in the k sweep)
    const double q1 = volhalf * (s[c] + s[c - sd]), q2 = volhalf * (s[N + c] + s[N + c - sd]), q3 = volhalf * (s[2 * N + c] + s[2 * N + c - sd]);
    const double u = b.w[N + c], v = b.w[2 * N + c], w = b.w[3 * N + c];
    const double q = q1 * u + q2 * v + q3 * w - 0.0;
    const double cijk = sqrt(c_prm.gammaInf * b.p[c] / rho);
    const double cs = cijk * sqrt(q1 * q1 + q2 * q2 + q3 * q3);
    const double r1 = volhalf * (s[c] + slow[c - sd]), r2 = volhalf * (s[N + c] + slow[N + c - sd]), r3 = volhalf * (s[2 * N + c] + slow[2 * N + c - sd]);
    const double eps2 = epsval * epsval * cInf2 * (r1 * r1 + r2 * r2 + r3 * r3);
    const double t0 = fac * sqrt(q * q + eps2), t1 = fac * sqrt((q + cs) * (q + cs) + eps2), t2 = fac * sqrt((q - cs) * (q - cs) + eps2);
    A.dP[0] = 0.5 * (q + t0); A.dP[1] = 0.5 * (q + cs + t1); A.dP[2] = 0.5 * (q - cs + t2);
    A.dM[0] = 0.5 * (q - t0); A.dM[1] = 0.5 * (q + cs - t1); A.dM[2] = 0.5 * (q - cs - t2);
    A.dtrb = (cfl * b.dtl[c] * vol) * dmax_((double)b.iblank[c], 0.0);
}

__device__ __forceinline__ void unit_half_sum(const double* __restrict__ ssum, int N, int c, double r[3], double& len) {
    r[0] = 0.5 * ssum[c]; r[1] = 0.5 * ssum[N + c]; r[2] = 0.5 * ssum[2 * N + c];
    len = sqrt(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]);
}

// incoming change of basis for cell c.  DIR 0 (j sweep): scale by -cfl*dtl*vol (smoothers.F90:520)
// and T_eta^-1; DIR 1 (i sweep): rotation (ri, rj); DIR 2 (k sweep): rotation (ri, rk).
template <int DIR>
__device__ __forceinline__ void dadi_pre(const BlockDev& b, int N, int c, double cfl, double f[5]) {
    double dw1 = f[0], dw2 = f[1], dw3 = f[2], dw4 = f[3], dw5 = f[4];
    if (DIR == 0) {
        const double dt = -cfl * b.dtl[c] * b.vol[c];
        dw1 *= dt; dw2 *= dt; dw3 *= dt; dw4 *= dt; dw5 *= dt;
        const double gam = c_prm.gammaInf, gm1 = gam - 1.0;
        const double rho = b.w[c], uvel = b.w[N + c], vvel = b.w[2 * N + c], wvel = b.w[3 * N + c];
        const double cijk = sqrt(gam * b.p[c] / rho);
        const double c2inv = 1.0 / (cijk * cijk);
        const double xfact = 2.0 * cijk;
        const double alphinv = sqrt(2.0) * cijk / rho;
        const double uvw = 0.5 * (uvel * uvel + vvel * vvel + wvel * wvel);
        double rj[3], len;
        unit_half_sum(b.ssum + 3 * N, N, c, rj, len);
        const double uu = uvel * rj[0] + vvel * rj[1] + wvel * rj[2];
        const double rj1 = rj[0] / len, rj2 = rj[1] / len, rj3 = rj[2] / len;
        double a1 = dw2 * uvel + dw3 * vvel + dw4 * wvel - dw5;
        a1 = a1 * gm1 * c2inv + dw1 * (1.0 - uvw * gm1 * c2inv);
        const double a2 = (rj2 * wvel - rj3 * vvel) * dw1 + rj3 * dw3 - rj2 * dw4;
        const double a3 = (rj3 * uvel - rj1 * wvel) * dw1 + rj1 * dw4 - rj3 * dw2;
        const double a4 = (rj1 * vvel - rj2 * uvel) * dw1 + rj2 * dw2 - rj1 * dw3;
        double a5 = uvw * dw1 - uvel * dw2 - vvel * dw3 - wvel * dw4 + dw5;
        a5 = a5 * gm1 * c2inv;
        const double a6 = uu * dw1 / len - rj1 * dw2 - rj2 * dw3 - rj3 * dw4;
        f[0] = a1 * rj1 + a2 / rho;
        f[1] = a1 * rj2 + a3 / rho;
        f[2] = a1 * rj3 + a4 / rho;
        f[3] = (0.5 * a5 - a6 / xfact) * alphinv;
        f[4] = (0.5 * a5 + a6 / xfact) * alphinv;
    } else {
        double ri[3], rx[3], li, lx;
        unit_half_sum(b.ssum, N, c, ri, li);
        unit_half_sum(b.ssum + (DIR == 1 ? 3 : 6) * N, N, c, rx, lx);
        ri[0] /= li; ri[1] /= li; ri[2] /= li;
        rx[0] /= lx; rx[1] /= lx; rx[2] /= lx;
        const double sqrt2inv = 1.0 / sqrt(2.0);
        const double a1 = ri[0] * rx[0] + ri[1] * rx[1] + ri[2] * rx[2];
        double a2, a3, a4;
        if (DIR == 1) {
            a2 = ri[0] * rx[1] - rx[0] * ri[1];
            a3 = ri[2] * rx[1] - rx[2] * ri[1];
            a4 = ri[0] * rx[2] - rx[0] * ri[2];
        } else {
            a2 = rx[0] * ri[1] - ri[0] * rx[1];
            a3 = rx[2] * ri[1] - ri[2] * rx[1];
            a4 = rx[0] * ri[2] - ri[0] * rx[2];
        }
        const double a5 = (dw4 - dw5) * sqrt2inv;
        const double a6 = (dw4 + dw5) * 0.5;
        const double a7 = (a3 * dw1 + a4 * dw2 - a2 * dw3 - a5 * a1) * sqrt2inv;
        f[0] = a1 * dw1 + a2 * dw2 + a4 * dw3 + a5 * a3;
        f[1] = -a2 * dw1 + a1 * dw2 - a3 * dw3 + a5 * a4;
        f[2] = -a4 * dw1 + a3 * dw2 + a1 * dw3 - a5 * a2;
        f[3] = -a7 + a6;
        f[4] = a7 + a6;
    }
}

// T_zeta back to conservative variables and the -1/vol scaling (residuals.F90:1679-1746)
__device__ __forceinline__ void dadi_post(const BlockDev& b, int N, int c, double f[5]) {
    const double gam = c_prm.gammaInf;
    const double rho = b.w[c], uvel = b.w[N + c], vvel = b.w[2 * N + c], wvel = b.w[3 * N + c];
    double rk[3], len;
    unit_half_sum(b.ssum + 6 * N, N, c, rk, len);
    const double uu = uvel * rk[0] + vvel * rk[1] + wvel * rk[2];
    const double rk1 = rk[0] / len, rk2 = rk[1] / len, rk3 = rk[2] / len;
    const double uvw = 0.5 * (uvel * uvel + vvel * vvel + wvel * wvel);
    const double cijkinv = sqrt(rho / gam / b.p[c]);
    const double alph = rho * cijkinv * (1.0 / sqrt(2.0));
    const double xfact = 2.0 / cijkinv;
    const double ge = gam * b.w[4 * N + c] / rho - (gam - 1.0) * uvw;
    const double dw1 = f[0], dw2 = f[1], dw3 = f[2], dw4 = f[3] * alph, dw5 = f[4] * alph;
    const double a1 = dw1 * rk1 + dw2 * rk2 + dw3 * rk3 + dw4 + dw5;
    const double a2 = 0.5 * xfact * (dw4 - dw5);
    const double a3 = uvw * (rk1 * dw1 + rk2 * dw2 + rk3 * dw3);
    const double volfact = -1.0 / b.vol[c];
    f[0] = a1 * volfact;
    f[1] = (a1 * uvel - rho * (rk3 * dw2 - rk2 * dw3) + a2 * rk1) * volfact;
    f[2] = (a1 * vvel - rho * (rk1 * dw3 - rk3 * dw1) + a2 * rk2) * volfact;
    f[3] = (a1 * wvel - rho * (rk2 * dw1 - rk1 * dw2) + a2 * rk3) * volfact;
    f[4] = (a3 + rho * ((vvel * rk3 - wvel * rk2) * dw1 + (wvel * rk1 - uvel * rk3) * dw2 + (uvel * rk2 - vvel * rk1) * dw3) +
            (ge + 0.5 * xfact * uu / len) * dw4 + (ge - 0.5 * xfact * uu / len) * dw5) * volfact;
}

// The sweep is split so that only the recurrence itself is serial:
//   k_dadi_coef   (one thread per cell)      : cell coefficients of the sweep direction -> work[0..8],
//                                              incoming change of basis applied to dw in place
//   k_dadi_thomas (one thread per line and variable): Thomas elimination / back substitution
//                                              (tridiagsolve, residuals.F90:1750-1783) reading only
//                                              the precomputed arrays
//   k_dadi_post   (one thread per cell, k sweep only): T_zeta and the -1/vol scaling
// `work` is the face-flux workspace b.flux (free while the smoother update runs): slots 0..8 cell
// coefficients, 9..13 the eliminated super-diagonal per variable, 14..18 the forward-swept rhs,
// 19..27 the tridiagonal rows per coefficient set (k_dadi_tri).
template <int DIR>
__global__ void __launch_bounds__(128) k_dadi_coef(Dims d, BlockDev b, int sd, double cfl) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N;
    const int c = i + (int)d.sJ * j + (int)d.sK * k;
    const bool viscous = c_prm.equations != ADFB_EULER, eddy = c_prm.equations == ADFB_RANS;
    const double* s = DIR == 0 ? b.sj : (DIR == 1 ? b.si : b.sk);
    const double* slow = DIR == 2 ? b.sj : s;  // reference quirk, residuals.F90:1625-1627
    DadiCoef A;
    dadi_cell(b, N, c, sd, s, slow, cfl, viscous, eddy, A);
    double* w = b.flux;
#pragma unroll
    for (int t = 0; t < 3; t++) { w[t * N + c] = A.dP[t]; w[(3 + t) * N + c] = A.dM[t]; }
    w[6 * N + c] = A.vt1; w[7 * N + c] = A.vt3; w[8 * N + c] = A.dtrb;
    double f[5];
#pragma unroll
    for (int n = 0; n < 5; n++) f[n] = b.dw[n * N + c];
    dadi_pre<DIR>(b, N, c, cfl, f);
#pragma unroll
    for (int n = 0; n < 5; n++) b.dw[n * N + c] = f[n];
}

__global__ void __launch_bounds__(128) k_dadi_post(Dims d, BlockDev b) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N;
    const int c = i + (int)d.sJ * j + (int)d.sK * k;
    double f[5];
#pragma unroll
    for (int n = 0; n < 5; n++) f[n] = b.dw[n * N + c];
    dadi_post(b, N, c, f);
#pragma unroll
    for (int n = 0; n < 5; n++) b.dw[n * N + c] = f[n];
}

// tridiagonal rows of the three coefficient sets from the cell coefficients of the cell and its two line
// neighbours (residuals.F90:1374-1391): work slots 19+t (diagonal), 22+t (sub-), 25+t (super-diagonal)
__global__ void __launch_bounds__(256) k_dadi_tri(Dims d, BlockDev b, int sd, int dirIdx) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N;
    const int c = i + (int)d.sJ * j + (int)d.sK * k;
    const int m = dirIdx == 0 ? j : (dirIdx == 1 ? i : k);
    const int l = dirIdx == 0 ? d.jl : (dirIdx == 1 ? d.il : d.kl);
    const double* w = b.flux;
    const double dt = w[8 * N + c];
    const double vt2 = w[6 * N + c] + w[7 * N + c];
#pragma unroll
    for (int t = 0; t < 3; t++) {
        b.flux[(19 + t) * N + c] = 1.0 + (vt2 + w[t * N + c] - w[(3 + t) * N + c]) * dt;
        b.flux[(22 + t) * N + c] = (m > 2) ? (-w[6 * N + c - sd] - w[t * N + c - sd]) * dt : 0.0;
        b.flux[(25 + t) * N + c] = (m < l) ? (-w[7 * N + c + sd] + w[(3 + t) * N + c + sd]) * dt : 0.0;
    }
}

// one thread = one grid line (nl owned cells along sd) of one variable n = blockIdx.z
__global__ void __launch_bounds__(64) k_dadi_thomas(Dims d, BlockDev b, int sd, int nl, int s1, int n1, int s2, int n2) {
    ADFB_PDL_SYNC();
    const int q1 = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int q2 = blockIdx.y + 2;
    if (q1 > n1 + 1 || q2 > n2 + 1) return;
    const int n = blockIdx.z;
    const int t = n < 3 ? 0 : n - 2;   // coefficient set: (u), (u+c), (u-c)
    const int N = (int)d.N;
    const int base = q1 * s1 + q2 * s2;
    const int l = nl + 1;
    if (nl <= 1) return;  // `if (jl > 2)` guards: no implicit solve (changes of basis done by k_dadi_coef / k_dadi_post)
    const double* __restrict__ ccA = b.flux + (19 + t) * N;
    const double* __restrict__ bbA = b.flux + (22 + t) * N;
    const double* __restrict__ dsA = b.flux + (25 + t) * N;
    double* __restrict__ dd = b.flux + (9 + n) * N;
    double* __restrict__ fo = b.flux + (14 + n) * N;
    double* __restrict__ f = b.dw + n * N;
    double ddp = 0.0, ffp = 0.0;
    // The recurrence is walked in chunks of CH cells: all loads (and the recurrence-independent
    // arithmetic) of a chunk are issued first, so their latencies overlap; only 1/(cc - bb*dd) and
    // the rhs update form the serial chain.
    constexpr int CH = 8;
    for (int m0 = 2; m0 <= l; m0 += CH) {
        double cc[CH], bb[CH], ds[CH], fv[CH];
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 + u;
            if (m <= l) { const int c = base + m * sd; cc[u] = ccA[c]; bb[u] = bbA[c]; ds[u] = dsA[c]; fv[u] = f[c]; }
        }
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 + u;
            if (m <= l) {
                const int c = base + m * sd;
                const double d0 = (m == 2) ? 1.0 / cc[u] : 1.0 / (cc[u] - bb[u] * ddp);
                const double ddm = ds[u] * d0;
                dd[c] = ddm;
                const double v = (m == 2) ? fv[u] * d0 : (fv[u] - bb[u] * ffp) * d0;
                fo[c] = v;
                ffp = v; ddp = ddm;
            }
        }
    }
    // back substitution; ffp holds ff(l)
    f[base + l * sd] = ffp;
    for (int m0 = l - 1; m0 >= 2; m0 -= CH) {
        double fr[CH], dr[CH];
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 - u;
            if (m >= 2) { const int c = base + m * sd; fr[u] = fo[c]; dr[u] = dd[c]; }
        }
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 - u;
            if (m >= 2) {
                const double v = fr[u] - dr[u] * ffp;
                f[base + m * sd] = v;
                ffp = v;
            }
        }
    }
}

// Tiled variant of k_dadi_thomas: one WARP = 32 neighbouring lines of one variable.  The recurrence is walked in chunks of
// ADFB_DT_CH cells; the operands of a chunk (tridiagonal rows, right-hand side) are staged as a [line][cell] tile in shared
// memory with cp.async, the next chunk's tile in flight while the current one is eliminated, and the results leave through a
// tile as well.  Two things are gained over the per-thread walk: (1) the load latency of a chunk is no longer serialised
// with the arithmetic of the previous one (12 dependent round trips per sweep on a 96-cell line), (2) for lines along i
// (sd == 1), where neighbouring THREADS own lines a whole row apart, the lanes copy along the line (8 consecutive cells =
// one 64-byte segment per 8 lanes) instead of touching 32 cache lines per load instruction -- that sweep was bound by L1
// wavefronts.  Same operations on the same operands.
#define ADFB_DT_CH 8
#define ADFB_DT_WARPS 4
struct DtSmem {
    double in[2][4][32][ADFB_DT_CH + 1];   // [stage][array][line][cell]; odd pitch: conflict-free 64-bit accesses down a column
    double out[2][32][ADFB_DT_CH + 1];
};
static const size_t kDadiTileSmem = sizeof(DtSmem) * ADFB_DT_WARPS;   // dynamic shared memory of one CTA
__device__ __forceinline__ void dt_cp8(double* dst, const double* src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void dt_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int NPEND>
__device__ __forceinline__ void dt_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(NPEND) : "memory"); }

__global__ void __launch_bounds__(32 * ADFB_DT_WARPS) k_dadi_thomas_tile(Dims d, BlockDev b, int sd, int nl, int s1, int n1, int s2, int n2) {
    ADFB_PDL_SYNC();
    constexpr int CH = ADFB_DT_CH;
    extern __shared__ __align__(16) unsigned char dt_raw[];
    DtSmem& S = reinterpret_cast<DtSmem*>(dt_raw)[threadIdx.x >> 5];
    const int lane = threadIdx.x & 31;
    const int groups = (n1 + 31) / 32;
    long long item = (long long)blockIdx.x * ADFB_DT_WARPS + (threadIdx.x >> 5);
    if (item >= (long long)groups * n2 * 5 || nl <= 1) return;   // whole warps leave; only __syncwarp below
    const int n = (int)(item % 5);
    item /= 5;
    const int grp = (int)(item % groups), q2 = (int)(item / groups) + 2;
    const int t = n < 3 ? 0 : n - 2;   // coefficient set: (u), (u+c), (u-c)
    const int N = (int)d.N;
    const int q10 = grp * 32 + 2;
    const int nLines = (n1 + 2 - q10) < 32 ? (n1 + 2 - q10) : 32;
    const int base0 = q10 * s1 + q2 * s2;
    const int l = nl + 1;
    const double* __restrict__ ccA = b.flux + (19 + t) * N;
    const double* __restrict__ bbA = b.flux + (22 + t) * N;
    const double* __restrict__ dsA = b.flux + (25 + t) * N;
    double* dd = b.flux + (9 + n) * N;
    double* fo = b.flux + (14 + n) * N;
    double* f = b.dw + n * N;
    const bool alongLine = sd == 1;
    const int nChunks = (nl + CH - 1) / CH;
    // The 32 x CH tile is copied by the warp in CH passes of 32 elements.  Lines along i (sd == 1): lane -> cell u = lane % CH of
    // line lane / CH + (32 / CH) * pass (8 lanes = one 64-byte segment of a line); otherwise lane -> line, pass -> cell (32 lanes =
    // 256 contiguous bytes across the lines).  Global and shared offsets of the passes are fixed per lane; a chunk adds m0 * sd.
    int gOff[CH], sOff[CH];
    unsigned okLine = 0;   // bit r: the line of pass r exists
#pragma unroll
    for (int r = 0; r < CH; r++) {
        const int ln = alongLine ? (lane / CH) + (32 / CH) * r : lane;
        const int u = alongLine ? lane % CH : r;
        gOff[r] = base0 + ln * s1 + u * sd;
        sOff[r] = ln * (CH + 1) + u;
        if (ln < nLines) okLine |= 1u << r;
    }
    const int uLane = alongLine ? lane % CH : 0;   // cell of the lane's elements (alongLine); pass index otherwise
    double* const in0 = &S.in[0][0][0][0];
    double* const out0 = &S.out[0][0][0];
    constexpr int TILE = 32 * (CH + 1);
    auto issueF = [&](int chunk, int stage) {
        const int m0 = 2 + chunk * CH;
        double* t0 = in0 + stage * 4 * TILE;
#pragma unroll
        for (int r = 0; r < CH; r++) {
            const int m = m0 + (alongLine ? uLane : r);
            if (((okLine >> r) & 1u) && m <= l) {
                const int c = gOff[r] + m0 * sd;
                dt_cp8(t0 + sOff[r], ccA + c);
                dt_cp8(t0 + TILE + sOff[r], bbA + c);
                dt_cp8(t0 + 2 * TILE + sOff[r], dsA + c);
                dt_cp8(t0 + 3 * TILE + sOff[r], f + c);
            }
        }
        dt_commit();
    };
    double ddp = 0.0, ffp = 0.0;
    issueF(0, 0);
    for (int ch = 0; ch < nChunks; ch++) {
        const int st = ch & 1;
        if (ch + 1 < nChunks) { issueF(ch + 1, st ^ 1); dt_wait<1>(); } else dt_wait<0>();
        __syncwarp();
        const int m0 = 2 + ch * CH;
        if (lane < nLines) {
#pragma unroll
            for (int u = 0; u < CH; u++) {
                const int m = m0 + u;
                if (m <= l) {
                    const double cc = S.in[st][0][lane][u], bb = S.in[st][1][lane][u], ds = S.in[st][2][lane][u], fv = S.in[st][3][lane][u];
                    const double d0 = (m == 2) ? 1.0 / cc : 1.0 / (cc - bb * ddp);
                    const double ddm = ds * d0;
                    S.out[0][lane][u] = ddm;
                    const double v = (m == 2) ? fv * d0 : (fv - bb * ffp) * d0;
                    S.out[1][lane][u] = v;
                    ffp = v; ddp = ddm;
                }
            }
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < CH; r++) {
            const int m = m0 + (alongLine ? uLane : r);
            if (((okLine >> r) & 1u) && m <= l) {
                const int c = gOff[r] + m0 * sd;
                dd[c] = out0[sOff[r]];
                fo[c] = out0[TILE + sOff[r]];
            }
        }
        __syncwarp();
    }
    // back substitution, chunks in reverse; ffp holds ff(l) = the value stored at m = l
    auto issueB = [&](int chunk, int stage) {
        const int m0 = 2 + chunk * CH;
        double* t0 = in0 + stage * 4 * TILE;
#pragma unroll
        for (int r = 0; r < CH; r++) {
            const int m = m0 + (alongLine ? uLane : r);
            if (((okLine >> r) & 1u) && m <= l) {
                const int c = gOff[r] + m0 * sd;
                dt_cp8(t0 + sOff[r], fo + c);
                dt_cp8(t0 + TILE + sOff[r], dd + c);
            }
        }
        dt_commit();
    };
    issueB(nChunks - 1, 0);
    for (int ch = nChunks - 1, it = 0; ch >= 0; ch--, it++) {
        const int st = it & 1;
        if (ch > 0) { issueB(ch - 1, st ^ 1); dt_wait<1>(); } else dt_wait<0>();
        __syncwarp();
        const int m0 = 2 + ch * CH;
        if (lane < nLines) {
#pragma unroll
            for (int u = CH - 1; u >= 0; u--) {
                const int m = m0 + u;
                if (m <= l) {
                    const double fr = S.in[st][0][lane][u], dr = S.in[st][1][lane][u];
                    const double v = (m == l) ? fr : fr - dr * ffp;
                    S.out[0][lane][u] = v;
                    ffp = v;
                }
            }
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < CH; r++) {
            const int m = m0 + (alongLine ? uLane : r);
            if (((okLine >> r) & 1u) && m <= l) f[gOff[r] + m0 * sd] = out0[sOff[r]];
        }
        __syncwarp();
    }
}

}  // namespace

// computedwDADI including the -cfl*dtl*vol scaling of executeDADIStep (smoothers.F90:515-528)
static int launch_dadi(const Dims& d, const BlockDev& b, const AdfbParams& prm, cudaStream_t s) {
    const int sJ = (int)d.sJ, sK = (int)d.sK;
    const dim3 tc(32, 4, 1);
    const dim3 gc((d.nx + 31) / 32, (d.ny + 3) / 4, d.nz);
    const dim3 tb(32, 1, 1);
    // (a partitioned, 8-lanes-per-line variant of this solve was measured slower here: with 5 systems per line the
    // serial walks already fill the machine and the partition method does 2.5x the arithmetic; it pays for the
    // single-system SA solve only, see sa_kernels.cuh)
    // i lines (sd == 1) take the tiled walk: in the per-thread walk neighbouring threads own lines a whole row apart
    auto thomas = [&](int sd, int nl, int s1, int n1, int s2, int n2) {
        if (sd == 1) {
            const long long items = (long long)((n1 + 31) / 32) * n2 * 5;
            cudaLaunchConfig_t cfg = {};
            cfg.gridDim = dim3((unsigned)((items + ADFB_DT_WARPS - 1) / ADFB_DT_WARPS)); cfg.blockDim = dim3(32 * ADFB_DT_WARPS);
            cfg.dynamicSmemBytes = kDadiTileSmem; cfg.stream = s;
            cudaLaunchAttribute attr[1];
            attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
            attr[0].val.programmaticStreamSerializationAllowed = 1;
            cfg.attrs = attr; cfg.numAttrs = 1;
            cudaLaunchKernelEx(&cfg, k_dadi_thomas_tile, d, b, sd, nl, s1, n1, s2, n2);
            return;
        }
        launch_pdl(k_dadi_thomas, dim3((n1 + 31) / 32, n2, 5), tb, s, d, b, sd, nl, s1, n1, s2, n2);
    };
    // rows + solve of one direction
    auto solve = [&](int sd, int dirIdx, int nl, int s1, int n1, int s2, int n2) {
        KT_BEGIN(K_DADI, s);
        launch_pdl(k_dadi_tri, gc, tc, s, d, b, sd, dirIdx);
        KT_END(K_DADI, s);
        KT_BEGIN(K_DADI, s);
        thomas(sd, nl, s1, n1, s2, n2);
        KT_END(K_DADI, s);
    };
    // j sweep
    KT_BEGIN(K_DADI, s);
    launch_pdl(k_dadi_coef<0>, gc, tc, s, d, b, sJ, prm.cfl);
    KT_END(K_DADI, s);
    solve(sJ, 0, d.ny, 1, d.nx, sK, d.nz);
    // i sweep
    KT_BEGIN(K_DADI, s);
    launch_pdl(k_dadi_coef<1>, gc, tc, s, d, b, 1, prm.cfl);
    KT_END(K_DADI, s);
    solve(1, 1, d.nx, sJ, d.ny, sK, d.nz);
    // k sweep
    KT_BEGIN(K_DADI, s);
    launch_pdl(k_dadi_coef<2>, gc, tc, s, d, b, sK, prm.cfl);
    KT_END(K_DADI, s);
    solve(sK, 2, d.nz, 1, d.nx, sJ, d.ny);
    KT_BEGIN(K_DADI, s);
    launch_pdl(k_dadi_post, gc, tc, s, d, b);
    KT_END(K_DADI, s);
    return (int)cudaGetLastError();
}
