// sa_kernels.cuh -- Spalart-Allmaras DD-ADI solve (turbSolveDDADI, src/turbulence/turbAPI.F90:4-95;
// sa_block / saSolve, src/turbulence/sa.F90:16-86, 717-1267)
//
//   k_sa_bmt    : bcTurbTreatment (turbBCRoutines.F90:662-797) for the scalar SA variable: the
//                 1x1 "matrix" bmt of every boundary face cell next to an owned cell, stored at
//                 its first-halo cell
//   k_sa_rhs    : block-path saSource (:89-344) + turbAdvection (turbUtils.F90:828-1553) +
//                 saViscous (:346-676) incl. the implicit diagonal qq; saResScale (:678-714)
//   k_sa_line   : one dd-ADI sweep: per grid line a scalar tridiagonal system (diffusion +
//                 first-order upwind advection off-diagonals, qq on the diagonal), eliminated
//                 backward then substituted forward exactly like the reference (:979-992)
//   k_sa_update : nuTilde += dvt, clip >= 0 (:1257-1262), saEddyViscosity on the owned cells
// scratch slots: 0 = dvt, 1 = qq, 2 = bmt, 3 = eliminated diagonal of the current sweep.
#pragma once
#include "adfb_common.cuh"
#include "tridiag_part.cuh"
#include "smoother_kernels.cuh"
#include <math.h>

namespace {

// The subfaces of the list in one launch (blockIdx.z = subface).  The values are read at the first-halo cells next to OWNED
// cells only (k_sa_rhs, k_sa_coef), so each subface is clipped to its owned in-plane range: no cell is written by two
// subfaces and the launch order of the reference's loop does not matter.
__global__ void __launch_bounds__(128) k_sa_bmt(Dims d, BlockDev b, const __grid_constant__ BcList L) {
    ADFB_PDL_SYNC();
    const int q = blockIdx.z;
    const FaceDev& f = L.f[q];
    const int a0 = f.icBeg > 2 ? f.icBeg : 2, a1 = f.icEnd < L.la[q] ? f.icEnd : L.la[q];
    const int b0 = f.jcBeg > 2 ? f.jcBeg : 2, b1 = f.jcEnd < L.lb[q] ? f.jcEnd : L.lb[q];
    const int ia = blockIdx.x * blockDim.x + threadIdx.x + a0;
    const int jb = blockIdx.y * blockDim.y + threadIdx.y + b0;
    if (ia > a1 || jb > b1) return;
    const long long N = d.N;
    const long long c1 = f.off[1] + ia * f.sa + jb * f.sb;
    const long long na = f.icEnd - f.icBeg + 1, nb = f.jcEnd - f.jcBeg + 1;
    const long long o = (ia - f.icBeg) + na * (jb - f.jcBeg);
    double bmt = -1.0;
    if (f.bcType == ADFB_BC_NSWALL_ADIABATIC || f.bcType == ADFB_BC_NSWALL_ISOTHERMAL || f.bcType == ADFB_BC_SUBSONIC_INFLOW ||
        f.bcType == ADFB_BC_SUPERSONIC_INFLOW) bmt = 1.0;   // bcTurbWall / bcTurbInflow
    else if (f.bcType == ADFB_BC_FARFIELD) {
        const double dot = f.norm[o] * c_prm.wInf[1] + f.norm[o + na * nb] * c_prm.wInf[2] + f.norm[o + 2 * na * nb] * c_prm.wInf[3] -
                           (f.rface ? f.rface[o] : 0.0);
        bmt = dot > 0.0 ? -1.0 : 0.0;
    }
    b.scratch[2 * N + c1] = bmt;
}

// diffusion coefficients of cell c along sd (shared by the residual and the line solve)
__device__ __forceinline__ void sa_diff_coef(const BlockDev& b, int N, int c, int sd, const double* __restrict__ s,
                                             const double* __restrict__ ssum, double nu, double& c1m, double& c1p,
                                             double& xa, double& ya, double& za) {
    const double* w = b.w;
    const double* vol = b.vol;
    const int cm = c - sd, cp = c + sd;
    const double cb3Inv = c_fheat[3] /* 1 / rsaCb3 */, cb2 = c_prm.rsaCb2;
    const double vc = vol[c];
    const double voli = 1.0 / vc;
    const double volmi = 2.0 / (vc + vol[cm]);
    const double volpi = 2.0 / (vc + vol[cp]);
    const double xm = s[cm] * volmi, ym = s[N + cm] * volmi, zm = s[2 * N + cm] * volmi;
    const double xp = s[c] * volpi, yp = s[N + c] * volpi, zp = s[2 * N + c] * volpi;
    xa = 0.5 * ssum[c] * voli; ya = 0.5 * ssum[N + c] * voli; za = 0.5 * ssum[2 * N + c] * voli;
    const double ttm = xm * xa + ym * ya + zm * za;
    const double ttp = xp * xa + yp * ya + zp * za;
    const double nt0 = w[5 * N + c], ntm = w[5 * N + cm], ntp = w[5 * N + cp];
    const double cnud = -cb2 * nt0 * cb3Inv;
    const double cam = ttm * cnud, cap = ttp * cnud;
    const double nutm = 0.5 * (ntm + nt0), nutp = 0.5 * (ntp + nt0);
    const double num = 0.5 * (b.rlv[cm] / w[cm] + nu);
    const double nup = 0.5 * (b.rlv[cp] / w[cp] + nu);
    const double cdm = (num + (1.0 + cb2) * nutm) * ttm * cb3Inv;
    const double cdp = (nup + (1.0 + cb2) * nutp) * ttp * cb3Inv;
    c1m = dmax_(cdm + cam, 0.0);
    c1p = dmax_(cdp + cap, 0.0);
}

__global__ void __launch_bounds__(128, 4) k_sa_rhs(Dims d, BlockDev b, double factor) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = i + sJ * j + sK * k;
    const double* w = b.w;
    const double* bmt = b.scratch + 2 * N;
    // ---- source (block path: no eps clip on the strain production, sa.F90:198-215) ----
    double gv[3][3];
#pragma unroll
    for (int v = 0; v < 3; v++) {
        const double* q = w + (1 + v) * N;
        const double qip = q[c + 1], qim = q[c - 1], qjp = q[c + sJ], qjm = q[c - sJ], qkp = q[c + sK], qkm = q[c - sK];
#pragma unroll
        for (int m = 0; m < 3; m++) {
            const int o = m * N;
            gv[v][m] = qip * b.si[o + c] - qim * b.si[o + c - 1] + qjp * b.sj[o + c] - qjm * b.sj[o + c - sJ] + qkp * b.sk[o + c] - qkm * b.sk[o + c - sK];
        }
    }
    const double fact = 0.25 / b.vol[c];
    double ss, strainMag2 = 0.0;
    if (c_prm.turbProd == ADFB_PROD_STRAIN) {
        const double sxx = 2.0 * fact * gv[0][0], syy = 2.0 * fact * gv[1][1], szz = 2.0 * fact * gv[2][2];
        const double sxy = fact * (gv[0][1] + gv[1][0]), sxz = fact * (gv[0][2] + gv[2][0]), syz = fact * (gv[1][2] + gv[2][1]);
        const double div2 = (2.0 * (1.0 / 3.0)) * ((sxx + syy + szz) * (sxx + syy + szz));
        strainMag2 = 2.0 * (sxy * sxy + sxz * sxz + syz * syz) + sxx * sxx + syy * syy + szz * szz;
        ss = sqrt(2.0 * strainMag2 - div2);
    } else {
        const double vortx = 2.0 * fact * (gv[2][1] - gv[1][2]), vorty = 2.0 * fact * (gv[0][2] - gv[2][0]), vortz = 2.0 * fact * (gv[1][0] - gv[0][1]);
        ss = sqrt(vortx * vortx + vorty * vorty + vortz * vortz);
    }
    const double cv13 = c_prm.rsaCv1 * c_prm.rsaCv1 * c_prm.rsaCv1;
    const double kar2Inv = c_fheat[4];   // 1 / rsaK**2
    const double cw3 = c_prm.rsaCw3;
    const double cw36 = (cw3 * cw3 * cw3) * (cw3 * cw3 * cw3);
    const double nut = w[5 * N + c];
    const double nu = b.rlv[c] / w[c];
    const double dwl = b.d2Wall[c];
    const double dist2Inv = 1.0 / (dwl * dwl);
    const double chi = nut / nu, chi2 = chi * chi, chi3 = chi * chi2;
    const double fv1 = chi3 / (chi3 + cv13);
    const double fv2 = 1.0 - chi / (1.0 + chi * fv1);
    const double ft2 = c_prm.useft2SA ? c_prm.rsaCt3 * exp(-c_prm.rsaCt4 * chi2) : 0.0;
    double sst = ss + nut * fv2 * kar2Inv * dist2Inv;
    if (c_prm.useRotationSA) sst = sst + c_prm.rsaCrot * dmin_(0.0, sqrt(2.0 * strainMag2));
    sst = dmax_(sst, 1.e-10);
    double rr = nut * kar2Inv * dist2Inv / sst;
    rr = dmin_(rr, 10.0);
    const double rr2 = rr * rr, rr6 = rr2 * rr2 * rr2;
    const double gg = rr + c_prm.rsaCw2 * (rr6 - rr);
    const double gg2 = gg * gg, gg6 = gg2 * gg2 * gg2;
    const double termFw = pow((1.0 + cw36) / (gg6 + cw36), 1.0 / 6.0);
    const double fwSa = gg * termFw;
    const double term1 = c_prm.approxSA ? 0.0 : c_prm.rsaCb1 * (1.0 - ft2) * ss;
    const double term2 = dist2Inv * (kar2Inv * c_prm.rsaCb1 * ((1.0 - ft2) * fv2 + ft2) - c_prm.rsaCw1 * fwSa);
    double dvt = (term1 + term2 * nut) * nut;
    const double dfv1 = 3.0 * chi2 * cv13 / ((chi3 + cv13) * (chi3 + cv13));
    const double dfv2 = (chi2 * dfv1 - 1.0) / (nu * ((1.0 + chi * fv1) * (1.0 + chi * fv1)));
    const double dft2 = -2.0 * c_prm.rsaCt4 * chi * ft2 / nu;
    const double drr = (1.0 - rr * (fv2 + nut * dfv2)) * kar2Inv * dist2Inv / sst;
    const double dgg = (1.0 - c_prm.rsaCw2 + 6.0 * c_prm.rsaCw2 * (rr2 * rr2 * rr)) * drr;
    const double dfw = (cw36 / (gg6 + cw36)) * termFw * dgg;
    double qq = -2.0 * term2 * nut - dist2Inv * nut * nut * (c_prm.rsaCb1 * kar2Inv * (dfv2 - ft2 * dfv2 - fv2 * dft2 + dft2) - c_prm.rsaCw1 * dfw);
    qq = dmax_(qq, 0.0);
    // ---- advection k, j, i (first/second order upwind) with the BC coupling of qq ----
    const double voli2 = 0.5 / b.vol[c];
    const double ux = w[N + c], uy = w[2 * N + c], uz = w[3 * N + c];
    const int sdv[3] = {1, sJ, sK};
    const int idx[3] = {i, j, k}, last[3] = {d.il, d.jl, d.kl};
    const double* nt = w + 5 * N;
#pragma unroll
    for (int a = 2; a >= 0; a--) {
        const int sd = sdv[a];
        const double* ssum = b.ssum + 3 * a * N;
        const double xa = ssum[c] * voli2, ya = ssum[N + c] * voli2, za = ssum[2 * N + c] * voli2;
        const double uu = xa * ux + ya * uy + za * uz;
        double dwtx;
        if (uu > 0.0) {
            if (c_prm.secondOrdTurb) {
                const double dwtm1 = nt[c - sd] - nt[c - 2 * sd], dwt = nt[c] - nt[c - sd], dwtp1 = nt[c + sd] - nt[c];
                dwtx = dwt;
                if (dwt * dwtp1 > 0.0) dwtx = dwtx + 0.5 * ((fabs(dwt) < fabs(dwtp1)) ? dwt : dwtp1);
                if (dwt * dwtm1 > 0.0) dwtx = dwtx - 0.5 * ((fabs(dwt) < fabs(dwtm1)) ? dwt : dwtm1);
            } else dwtx = nt[c] - nt[c - sd];
            dvt = dvt - uu * dwtx;
            qq = qq + uu;
            if (idx[a] == 2) qq = qq + uu * dmax_(bmt[c - sd], 0.0);
        } else {
            if (c_prm.secondOrdTurb) {
                const double dwtm1 = nt[c] - nt[c - sd], dwt = nt[c + sd] - nt[c], dwtp1 = nt[c + 2 * sd] - nt[c + sd];
                dwtx = dwt;
                if (dwt * dwtp1 > 0.0) dwtx = dwtx - 0.5 * ((fabs(dwt) < fabs(dwtp1)) ? dwt : dwtp1);
                if (dwt * dwtm1 > 0.0) dwtx = dwtx + 0.5 * ((fabs(dwt) < fabs(dwtm1)) ? dwt : dwtm1);
            } else dwtx = nt[c + sd] - nt[c];
            dvt = dvt - uu * dwtx;
            qq = qq - uu;
            if (idx[a] == last[a]) qq = qq - uu * dmax_(bmt[c + sd], 0.0);
        }
    }
    // ---- diffusion k, j, i ----
#pragma unroll
    for (int a = 2; a >= 0; a--) {
        const int sd = sdv[a];
        const double* s = a == 0 ? b.si : (a == 1 ? b.sj : b.sk);
        double c1m, c1p, xa, ya, za;
        sa_diff_coef(b, N, c, sd, s, b.ssum + 3 * a * N, nu, c1m, c1p, xa, ya, za);
        const double c10 = c1m + c1p;
        dvt = dvt + c1m * nt[c - sd] - c10 * nt[c] + c1p * nt[c + sd];
        if (idx[a] == 2) qq = qq + c10 - (-c1m) * dmax_(bmt[c - sd], 0.0);
        else if (idx[a] == last[a]) qq = qq + c10 - (-c1p) * dmax_(bmt[c + sd], 0.0);
        else qq = qq + c10;
    }
    const double rblank = dmax_((double)b.iblank[c], 0.0);
    b.dw[5 * N + c] = -b.volRef[c] * dvt * rblank;  // saResScale
    b.scratch[c] = dvt;
    b.scratch[N + c] = factor * qq;                 // saSolve :853-866 (implicit relaxation)
}

// one dd-ADI sweep along sd (saSolve, sa.F90:868-1255), split so that only the recurrence is serial:
//   k_sa_coef   (one thread per cell): off-diagonals bb, dd (diffusion + first-order upwind advection)
//               and the rhs ff = dvt * rblank  -> workspace b.flux slots 0..2
//   k_sa_thomas (one thread per line): backward elimination m = l..2 and forward substitution
//               (:979-998) reading only precomputed arrays; eliminated diagonal / rhs in slots 3, 4
__global__ void __launch_bounds__(128) k_sa_coef(Dims d, BlockDev b, int axis, int sd) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N;
    const int c = i + (int)d.sJ * j + (int)d.sK * k;
    const double* s = axis == 0 ? b.si : (axis == 1 ? b.sj : b.sk);
    const double* ssum = b.ssum + 3 * axis * N;
    const double nu = b.rlv[c] / b.w[c];
    double c1m, c1p, xa, ya, za;
    sa_diff_coef(b, N, c, sd, s, ssum, nu, c1m, c1p, xa, ya, za);
    double bb = -c1m, dd = -c1p;
    const double uu = xa * b.w[N + c] + ya * b.w[2 * N + c] + za * b.w[3 * N + c];
    const double um = uu < 0.0 ? uu : 0.0, up = uu > 0.0 ? uu : 0.0;
    bb = bb - up;
    dd = dd + um;
    const double rblank = dmax_((double)b.iblank[c], 0.0);
    b.flux[c] = bb * rblank;
    b.flux[N + c] = dd * rblank;
    b.flux[2 * N + c] = b.scratch[c] * rblank;
}

__global__ void __launch_bounds__(64) k_sa_thomas(Dims d, BlockDev b, int sd, int nl, int s1, int n1, int s2, int n2, int multiplyByQQ) {
    ADFB_PDL_SYNC();
    const int q1 = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int q2 = blockIdx.y + 2;
    if (q1 > n1 + 1 || q2 > n2 + 1) return;
    const int N = (int)d.N;
    const int base = q1 * s1 + q2 * s2;
    const double* __restrict__ bbA = b.flux;
    const double* __restrict__ ddA = b.flux + N;
    const double* __restrict__ ffA = b.flux + 2 * N;
    double* __restrict__ ccO = b.flux + 3 * N;
    double* __restrict__ ffO = b.flux + 4 * N;
    const double* __restrict__ qq = b.scratch + N;
    double* __restrict__ dvt = b.scratch;
    const int l = nl + 1;
    // backward elimination m = l .. 2 (row l is untouched by it)
    double ccp = 0.0, ffp = 0.0, bbp = 0.0;
    constexpr int CH = 8;   // chunked walk: loads of a chunk first (latencies overlap), then the serial chain
    for (int m0 = l; m0 >= 2; m0 -= CH) {
        double cq[CH], fq[CH], bq[CH], dq[CH];
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 - u;
            if (m >= 2) { const int c = base + m * sd; cq[u] = qq[c]; fq[u] = ffA[c]; bq[u] = bbA[c]; dq[u] = ddA[c]; }
        }
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 - u;
            if (m >= 2) {
                const int c = base + m * sd;
                double cc = cq[u], ff = fq[u];
                if (m < l) {
                    const double f = dq[u] / ccp;
                    cc = cc - f * bbp;
                    ff = ff - f * ffp;
                }
                ccO[c] = cc; ffO[c] = ff;
                ccp = cc; ffp = ff; bbp = bq[u];
            }
        }
    }
    // forward substitution
    double xm = 0.0;
    for (int m0 = 2; m0 <= l; m0 += CH) {
        double fq[CH], bq[CH], cq[CH], qv[CH];
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 + u;
            if (m <= l) { const int c = base + m * sd; fq[u] = ffO[c]; bq[u] = bbA[c]; cq[u] = ccO[c]; qv[u] = qq[c]; }
        }
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int m = m0 + u;
            if (m <= l) {
                double ff = fq[u];
                if (m > 2) ff = ff - bq[u] * xm;
                ff = ff / cq[u];
                xm = ff;
                dvt[base + m * sd] = multiplyByQQ ? ff * qv[u] : ff;
            }
        }
    }
}

// the same sweep with every line spread over P lanes (tridiag_part.cuh); LS = 32 / P lines per warp
template <int P, int M>
__global__ void __launch_bounds__(32) k_sa_thomas_part(Dims d, BlockDev b, int sd, int nl, int s1, int n1, int s2, int n2, int multiplyByQQ) {
    ADFB_PDL_SYNC();
    typedef PartThomas<P, M> PT;
    const int lane = threadIdx.x, p = lane / PT::LS, lw = lane % PT::LS;
    int line = blockIdx.x * PT::LS + lw;
    const bool valid = line < n1 * n2;
    if (!valid) line = n1 * n2 - 1;  // every lane takes part in the shuffles; surplus lanes redo the last line
    const int N = (int)d.N;
    const int base = (line % n1 + 2) * s1 + (line / n1 + 2) * s2;
    const double* __restrict__ bbA = b.flux;
    const double* __restrict__ ddA = b.flux + N;
    const double* __restrict__ ffA = b.flux + 2 * N;
    const double* __restrict__ qq = b.scratch + N;
    double* __restrict__ dvt = b.scratch;
    int start, m;
    PT::chunk(nl, p, start, m);
    double ra[M], rb[M], rc[M], rd[M];
#pragma unroll
    for (int t = 0; t < M; t++) {
        ra[t] = 0.0; rb[t] = 1.0; rc[t] = 0.0; rd[t] = 0.0;
        if (t < m) {
            const int c = base + (2 + start + t) * sd;
            ra[t] = (start + t > 0) ? bbA[c] : 0.0;
            rb[t] = qq[c];
            rc[t] = (start + t < nl - 1) ? ddA[c] : 0.0;
            rd[t] = ffA[c];
        }
    }
    PT::solve(ra, rb, rc, rd, m, p, lw);
    if (!valid) return;
#pragma unroll
    for (int t = 0; t < M; t++) {
        if (t < m) {
            const int c = base + (2 + start + t) * sd;
            dvt[c] = multiplyByQQ ? rd[t] * qq[c] : rd[t];
        }
    }
}

__global__ void __launch_bounds__(256) k_sa_update(Dims d, BlockDev b) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N;
    const int c = i + (int)d.sJ * j + (int)d.sK * k;
    double nt = b.w[5 * N + c] + 1.0 * b.scratch[c];
    nt = dmax_(nt, 0.0);
    b.w[5 * N + c] = nt;
    const double rnuSA = nt * b.w[c];
    const double chi = rnuSA / b.rlv[c];
    const double chi3 = chi * chi * chi;
    const double cv13 = c_prm.rsaCv1 * c_prm.rsaCv1 * c_prm.rsaCv1;
    b.rev[c] = chi3 / (chi3 + cv13) * rnuSA;
}

}  // namespace

// sa_block(.false.) on one block
static int launch_sa_block(const Dims& d, const BlockDev& b, const AdfbParams& prm, const std::vector<AdfbSubface>& subs, cudaStream_t s) {
    const int sJ = (int)d.sJ, sK = (int)d.sK;
    cudaMemsetAsync(b.scratch + 2 * d.N, 0, sizeof(double) * d.N, s);
    for (size_t q0 = 0; q0 < subs.size(); q0 += ADFB_BC_MAXSUB) {
        const BcList L = make_bc_list(d, subs, q0);
        int ma = 1, mb = 1;
        for (int q = 0; q < L.n; q++) { ma = std::max(ma, L.f[q].icEnd - L.f[q].icBeg + 1); mb = std::max(mb, L.f[q].jcEnd - L.f[q].jcBeg + 1); }
        launch_kernel(K_SASOLVE, true, dim3((ma + 31) / 32, (mb + 3) / 4, (unsigned)L.n), dim3(32, 4), 0, s, k_sa_bmt, d, b, L);
    }
    const double factor = 1.0 + (1.0 - prm.alfaTurb) / prm.alfaTurb;
    {
        dim3 tr(32, 4, 1);
        dim3 g((d.nx + 31) / 32, (d.ny + 3) / 4, d.nz);
        launch_kernel(K_SASOLVE, true, g, tr, 0, s, k_sa_rhs, d, b, factor);
    }
    const dim3 tl(32, 1), tc(32, 4, 1), gc((d.nx + 31) / 32, (d.ny + 3) / 4, d.nz);
    auto sweep = [&](int axis, int sd, int nl, int s1, int n1, int s2, int n2, int mult) {
        launch_kernel(K_SASOLVE, true, gc, tc, 0, s, k_sa_coef, d, b, axis, sd);
        const int part = adfb_part_lanes(nl);
        if (part == 8 && nl <= 96) launch_kernel(K_SASOLVE, true, (n1 * n2 + 3) / 4, 32, 0, s, k_sa_thomas_part<8, 12>, d, b, sd, nl, s1, n1, s2, n2, mult);
        else if (part == 8) launch_kernel(K_SASOLVE, true, (n1 * n2 + 3) / 4, 32, 0, s, k_sa_thomas_part<8, 16>, d, b, sd, nl, s1, n1, s2, n2, mult);
        else if (part == 16) launch_kernel(K_SASOLVE, true, (n1 * n2 + 1) / 2, 32, 0, s, k_sa_thomas_part<16, 16>, d, b, sd, nl, s1, n1, s2, n2, mult);
        else launch_kernel(K_SASOLVE, true, dim3((n1 + 31) / 32, n2), tl, 0, s, k_sa_thomas, d, b, sd, nl, s1, n1, s2, n2, mult);
    };
    sweep(1, sJ, d.ny, 1, d.nx, sK, d.nz, 1);   // j lines
    sweep(0, 1, d.nx, sJ, d.ny, sK, d.nz, 1);   // i lines
    sweep(2, sK, d.nz, 1, d.nx, sJ, d.ny, 0);   // k lines
    {
        dim3 tb(32, 4, 2);
        dim3 g((d.nx + 31) / 32, (d.ny + 3) / 4, (d.nz + 1) / 2);
        launch_kernel(K_SASOLVE, true, g, tb, 0, s, k_sa_update, d, b);
    }
    if (launch_bc_levels(d, b, subs, 1, 1, 0, s)) return 1;
    return (int)cudaGetLastError();
}
