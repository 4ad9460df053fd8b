// residual_kernels.cuh -- residual kernels (face-flux form) for sm_90a
//
// Replaces the per-block residual core of the reference
// (blocketteResCore, src/NKSolver/blockette.F90:299-753 and its operator twins in
// src/solver/fluxes.F90, src/turbulence/sa.F90, src/utils/flowUtils.F90).
//
// The reference scatters every face flux to its two cells (`dw(i+1) -= fs; dw(i) += fs`).
// Here each face flux is computed exactly ONCE by the thread that owns the cell on the
// low side of the face (k_faces: the i+, j+ and k+ faces of cell c), stored in a face
// array, and k_div gathers the six faces of every owned cell in the order in which the
// reference's i/j/k sweeps touch that cell.  No atomics, no halo writes, results
// independent of launch geometry.
//
// Launch plan per residual evaluation (DESIGN.md section 4):
//   k_prep   : box cells  -> ss (entropy), aa, radI/J/K, [dtl]
//   k_nodal  : cells 1:ie -> dss(3); nodes 1:il -> 12 nodal gradients
//   k_faces  : cells 1:il x 1:jl x 1:kl -> central - JST - viscous flux of the 3 plus faces
//   k_div    : owned cells -> SA source/advection/diffusion row + flux divergence -> dw
//
// All index arithmetic is 32 bit (a block box times 30 components stays far below 2^31).
#pragma once
#include "adfb_common.cuh"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include "fused_kernels.cuh"
#include "geom_cell.cuh"

// tunables: threads per block / min resident blocks per SM
#ifndef FACES_TPB
#define FACES_TPB 128
#endif
#ifndef FACES_MINB
#define FACES_MINB 4
#endif
#ifndef FACES_MINB_SPLIT
#define FACES_MINB_SPLIT 6
#endif
#ifndef SA_TPB
#define SA_TPB 128
#endif
#ifndef SA_MINB
#define SA_MINB 6
#endif
#ifndef NODAL_TPB
#define NODAL_TPB 256
#endif
#ifndef NODAL_MINB
#define NODAL_MINB 1
#endif

#define IRHO 0
#define IVX 1
#define IVY 2
#define IVZ 3
#define IRHOE 4
#define ITU1 5

namespace {

// ---------------------------------------------------------------------------
// k_geom: geometry-derived static arrays (geom_cell.cuh), once per mesh (adfb_block_set_geometry)
__global__ void __launch_bounds__(256) k_geom(Dims d, BlockDev b) {
    geom_cell(d, b, blockIdx.x * blockDim.x + threadIdx.x, blockIdx.y * blockDim.y + threadIdx.y, blockIdx.z * blockDim.z + threadIdx.z);
}

// ---------------------------------------------------------------------------
// k_prep: entropy (inviscidDissFluxScalar, blockette.F90:3055-3089), speed of sound squared
// (:5168-5203), spectral radii and local time step (timeStep, :1899-2148).
// kOff / kTop: the planes kOff .. kTop only (slab pipeline of adfb_form_function); 0 / INT_MAX: all of them
// disc: the discretisation of the residual that reads ss (residual_discr); scaleRad: directional scaling of the radii
// (doScaling of timeStep: always on the blockette path, dirScaling .and. currentLevel <= groundLevel on the block path)
__global__ void __launch_bounds__(256) k_prep(Dims d, BlockDev b, int updateDt, int doRad, int kOff, int kTop, int disc, int scaleRad) {
    ADFB_PDL_SYNC();  // launched with programmatic stream serialization (launch_pdl)
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int j = blockIdx.y * blockDim.y + threadIdx.y;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + kOff;
    if (i > d.ib || j > d.jb || k > d.kb || k > kTop) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = i + sJ * j + sK * k;
    const double gam = c_prm.gammaInf;
    const double rho = b.w[c], p = b.p[c];
    // p / rho**gamma as p*exp(-gamma*log(rho)): |gamma*log(rho)| = O(1), so the result agrees
    // with pow() to a few ulp at less than half the FP64 instructions
    if (disc == ADFB_DISS_SCALAR) b.ss[c] = (c_prm.equations == ADFB_EULER) ? p : p * exp(-gam * log(rho));
    if (i < 1 || i > d.ie || j < 1 || j > d.je || k < 1 || k > d.ke) return;
    const bool viscous = c_prm.equations != ADFB_EULER;
    if (viscous) b.aa[c] = gam * p / rho;
    if (!doRad) return;  // smoother path: radii/dtl are frozen between timeStep calls

    const double clim2 = c_fheat[8];   // 0.000001 * gam * pInfCorr / rhoInf
    const double adis = c_prm.adis, asf = c_prm.acousticScaleFactor;
    const double ux = b.w[N + c], uy = b.w[2 * N + c], uz = b.w[3 * N + c];
    double cc2 = gam * p / rho;
    cc2 = dmax_(cc2, clim2);
    const double* ss = b.ssum;
    const double sxi = ss[c], syi = ss[N + c], szi = ss[2 * N + c];
    const double sxj = ss[3 * N + c], syj = ss[4 * N + c], szj = ss[5 * N + c];
    const double sxk = ss[6 * N + c], syk = ss[7 * N + c], szk = ss[8 * N + c];
    const double s2i = sxi * sxi + syi * syi + szi * szi;
    const double s2j = sxj * sxj + syj * syj + szj * szj;
    const double s2k = sxk * sxk + syk * syk + szk * szk;
    double ri = 0.5 * (fabs(ux * sxi + uy * syi + uz * szi) + asf * sqrt(cc2 * s2i));
    double rj = 0.5 * (fabs(ux * sxj + uy * syj + uz * szj) + asf * sqrt(cc2 * s2j));
    double rk = 0.5 * (fabs(ux * sxk + uy * syk + uz * szk) + asf * sqrt(cc2 * s2k));
    double dt = ri + rj + rk;
    if (!scaleRad) {   // doScaling = dirScaling .and. currentLevel <= groundLevel (solverUtils.F90:106)
        b.radI[c] = ri; b.radJ[c] = rj; b.radK[c] = rk;
    } else {
    ri = dmax_(ri, 1.e-25); rj = dmax_(rj, 1.e-25); rk = dmax_(rk, 1.e-25);
    // (ri/rj)**adis etc. via three logs and three exps (|adis*log(ratio)| < 10: error < 1e-15)
    const double li = log(ri), lj = log(rj), lk = log(rk);
    // (ri/rk)**adis = (ri/rj)**adis * (rj/rk)**adis: two exps instead of three (one more rounding, 1e-16)
    const double rij = exp(adis * (li - lj)), rjk = exp(adis * (lj - lk)), rik = rij * rjk;
    b.radI[c] = ri * (1.0 + 1.0 / rij + 1.0 / rik);
    b.radJ[c] = rj * (1.0 + 1.0 / rjk + rij);
    b.radK[c] = rk * (1.0 + rik + rjk);
    }

    if (!updateDt) return;
    if (i < 2 || i > d.il || j < 2 || j > d.jl || k < 2 || k > d.kl) return;
    if (viscous) {
        double rmu = b.rlv[c];
        rmu = rmu + b.rev[c];
        rmu = 0.5 * rmu / (rho * b.vol[c]);
        dt = dt + rmu * s2i;
        dt = dt + rmu * s2j;
        dt = dt + rmu * s2k;
    }
    const double plim = 0.001 * c_prm.pInfCorr;
    const double* pp = b.p;
    const double dpi = fabs(pp[c + 1] - 2.0 * p + pp[c - 1]) / (pp[c + 1] + 2.0 * p + pp[c - 1] + plim);
    const double dpj = fabs(pp[c + sJ] - 2.0 * p + pp[c - sJ]) / (pp[c + sJ] + 2.0 * p + pp[c - sJ] + plim);
    const double dpk = fabs(pp[c + sK] - 2.0 * p + pp[c - sK]) / (pp[c + sK] + 2.0 * p + pp[c - sK] + plim);
    const double rfl = 1.0 / (1.0 + 2.0 * (dpi + dpj + dpk));
    b.dtl[c] = rfl / dt;
}

// parameter-only constants evaluated once per adfb_set_params with the device's own arithmetic (c_fheat[2])
__global__ void k_param_consts(double* out) {
    out[0] = ff_sslim_eval(c_prm);
    // bcFarfield (BCRoutines.F90:1282-1396): free-stream entropy measure and speed of sound
    const double gam = c_prm.gammaInf;
    const double r0 = 1.0 / c_prm.wInf[0];
    out[1] = pow(c_prm.wInf[0], gam) / c_prm.pInfCorr;
    out[2] = sqrt(gam * c_prm.pInfCorr * r0);
}

// ---------------------------------------------------------------------------
// k_nodal: shock sensor dss (blockette.F90:3091-3105) on cells 1:ie and the nodal gradients
// (allNodalGradients, :5205-5515) on nodes 1:il in gather form.  For node n (= cell index c)
// the reference's three scatter sweeps add, in this order:  -K(layer k) +K(layer k+1)
// -J(layer j) +J(layer j+1) -I(layer i) +I(layer i+1), then scale by 1/(8 vol).
// GAOS (experiment switch ADFB_GRAD_AOS=1, main residual path only): the 12 gradients of a node are stored
// contiguously (96 B) and read back by k_faces with six 128-bit loads per node instead of twelve 64-bit ones
template <bool GAOS>
__global__ void __launch_bounds__(NODAL_TPB, NODAL_MINB) k_nodal(Dims d, BlockDev b, int doGrad, int dissApprox, int disc) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 1;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 1;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 1;
    if (i > d.ie || j > d.je || k > d.ke) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = i + sJ * j + sK * k;
    if (disc == ADFB_DISS_SCALAR) {
        const double sslim = c_fheat[2];   // 0.001 pInfCorr / rhoInf**gamma (pInfCorr for Euler), k_param_consts
        const double* ss = dissApprox ? b.shock : b.ss;  // *Approx: frozen sensor field (blockette.F90:4385-4396)
        const double s0 = ss[c];
        b.dss[c] = fabs((ss[c + 1] - 2.0 * s0 + ss[c - 1]) / (ss[c + 1] + 2.0 * s0 + ss[c - 1] + sslim));
        b.dss[N + c] = fabs((ss[c + sJ] - 2.0 * s0 + ss[c - sJ]) / (ss[c + sJ] + 2.0 * s0 + ss[c - sJ] + sslim));
        b.dss[2 * N + c] = fabs((ss[c + sK] - 2.0 * s0 + ss[c - sK]) / (ss[c + sK] + 2.0 * s0 + ss[c - sK] + sslim));
    } else if (disc == ADFB_DISS_MATRIX) {
        // pressure sensor with the omega blend, inviscidDissFluxMatrix blockette.F90:2495-2512
        const double plim = 0.001 * c_prm.pInfCorr;
        const double* p = dissApprox ? b.shock : b.p;  // matrix *Approx uses the frozen sensor (blockette.F90:4655-4670)
        const double p0 = p[c];
        const int sdv[3] = {1, sJ, sK};
#pragma unroll
        for (int m = 0; m < 3; m++) {
            const double pp = p[c + sdv[m]], pm = p[c - sdv[m]];
            b.dss[m * N + c] = fabs((pp - 2.0 * p0 + pm) / (0.5 * (pp + 2.0 * p0 + pm) + 0.5 * (fabs(pp - p0) + fabs(p0 - pm)) + plim));
        }
    }
    if (!doGrad || i > d.il || j > d.jl || k > d.kl) return;
    // the 8 cells around the node: bit0 = +i, bit1 = +j, bit2 = +k
    double q[8][4];
#pragma unroll
    for (int m = 0; m < 8; m++) {
        const int cc = c + (m & 1) + ((m >> 1) & 1) * sJ + ((m >> 2) & 1) * sK;
        q[m][0] = b.w[N + cc]; q[m][1] = b.w[2 * N + cc]; q[m][2] = b.w[3 * N + cc]; q[m][3] = b.aa[cc];
    }
    double g[12];
#pragma unroll
    for (int m = 0; m < 12; m++) g[m] = 0.0;
    // dir K: layers c (cells 0,1,2,3) and c+sK (4,5,6,7); J: (0,1,4,5) and (2,3,6,7); I: (0,2,4,6) and (1,3,5,7)
    const int lo[3][4] = {{0, 2, 4, 6}, {0, 1, 4, 5}, {0, 1, 2, 3}};
    const int hi[3][4] = {{1, 3, 5, 7}, {2, 3, 6, 7}, {4, 5, 6, 7}};
    const int sd[3] = {1, sJ, sK};
#pragma unroll
    for (int dd = 2; dd >= 0; dd--) {  // K, J, I
        const double* sv = b.sv + (3 * dd) * N;
#pragma unroll
        for (int side = 0; side < 2; side++) {
            const int* sel = side ? hi[dd] : lo[dd];
            const int cs = side ? c + sd[dd] : c;
            const double s1 = sv[cs], s2 = sv[N + cs], s3 = sv[2 * N + cs];
            double bar[4];
#pragma unroll
            for (int v = 0; v < 4; v++) bar[v] = 0.25 * (q[sel[0]][v] + q[sel[1]][v] + q[sel[2]][v] + q[sel[3]][v]);
            const double sg = side ? 1.0 : -1.0;
#pragma unroll
            for (int v = 0; v < 3; v++) {
                g[3 * v + 0] += sg * (bar[v] * s1);
                g[3 * v + 1] += sg * (bar[v] * s2);
                g[3 * v + 2] += sg * (bar[v] * s3);
            }
            g[9] -= sg * (bar[3] * s1);
            g[10] -= sg * (bar[3] * s2);
            g[11] -= sg * (bar[3] * s3);
        }
    }
    const double oVol = b.ovol[c];
    if (GAOS) {
        double2* o = reinterpret_cast<double2*>(b.grad + (long long)c * 12);
#pragma unroll
        for (int m = 0; m < 6; m++) o[m] = make_double2(g[2 * m] * oVol, g[2 * m + 1] * oVol);
    } else {
#pragma unroll
        for (int m = 0; m < 12; m++) b.grad[m * N + c] = g[m] * oVol;
    }
}

// ---------------------------------------------------------------------------
// one face of direction sd: central (inviscidCentralFlux, blockette.F90:2150-2428), scalar
// JST (inviscidDissFluxScalar, :3133-3338) and viscous (viscousFlux, :5576-6400) fluxes.
// c is the low-side cell, cp = c + sd.  Outputs fc[5] (central: dw(cp) -= fc, dw(c) += fc) and
// fd[5] = JST + viscous flux (the part the reference accumulates in fw with the same sign
// pattern for both: fw(cp) += f, fw(c) -= f).
struct CellState { double r, u, v, w, e, p; };

__device__ __forceinline__ CellState load_cell(const BlockDev& b, int N, int c) {
    CellState s;
    s.r = b.w[c]; s.u = b.w[N + c]; s.v = b.w[2 * N + c]; s.w = b.w[3 * N + c]; s.e = b.w[4 * N + c]; s.p = b.p[c];
    return s;
}

// APPROX bit 0: first-order/lumped dissipation (*Approx routines), bit 1: thin-layer viscous flux,
// bit 2: first-order coarse-level scalar dissipation (inviscidDissFluxScalarCoarse, fluxes.F90:4977-5203)
// PART: 0 = everything, 1 = central + dissipation only, 2 = viscous flux only (split launch, ADFB_SPLIT_FACES)
template <bool VISCOUS, int DISC, int APPROX, int PART = 0, bool GAOS = false>
__device__ __forceinline__ void face_flux(const BlockDev& b, int N, int c, int sd, int t1, int t2, int dir,
                                          const double* __restrict__ s, int8_t por, const double* __restrict__ rad,
                                          const double* __restrict__ dss, const CellState& m, double rFil, int doDiss,
                                          int doVisc, double fc[5], double fd[5], double* tq = nullptr) {
    const int cp = c + sd;
    const CellState q = load_cell(b, N, cp);
    const double s1 = s[c], s2 = s[N + c], s3 = s[2 * N + c];
    if (PART != 2) {   // central
        double vnp = q.u * s1 + q.v * s2 + q.w * s3;
        double vnm = m.u * s1 + m.v * s2 + m.w * s3;
        double porVel = 1.0, porFlux = 0.5;
        if (por == ADFB_NOFLUX) porFlux = 0.0;
        if (por == ADFB_BOUNDFLUX) { porVel = 0.0; vnp = 0.0; vnm = 0.0; }
        porVel = porVel * porFlux;
        const double qsp = vnp * porVel, qsm = vnm * porVel;
        const double rqsp = qsp * q.r, rqsm = qsm * m.r;
        const double pa = porFlux * (q.p + m.p);
        fc[0] = rqsp + rqsm;
        fc[1] = rqsp * q.u + rqsm * m.u + pa * s1;
        fc[2] = rqsp * q.v + rqsm * m.v + pa * s2;
        fc[3] = rqsp * q.w + rqsm * m.w + pa * s3;
        fc[4] = qsp * q.e + qsm * m.e + porFlux * (vnp * q.p + vnm * m.p);
    }
#pragma unroll
    for (int l = 0; l < 5; l++) fd[l] = 0.0;
    if (PART == 2) doDiss = 0;
    if (PART == 1) doVisc = 0;
    if (DISC == ADFB_DISS_SCALAR && (APPROX & 4) && doDiss) {
        const double ppor = (por == ADFB_NORMALFLUX) ? 0.5 : 0.0;
        const double dis0 = rFil * c_prm.vis2Coarse * ppor * (rad[c] + rad[cp]);
        fd[0] = dis0 * (q.r - m.r);
        fd[1] = dis0 * (q.u * q.r - m.u * m.r);
        fd[2] = dis0 * (q.v * q.r - m.v * m.r);
        fd[3] = dis0 * (q.w * q.r - m.w * m.r);
        fd[4] = dis0 * ((q.e + q.p) - (m.e + m.p));
    }
    if (DISC == ADFB_DISS_SCALAR && !(APPROX & 5) && doDiss) {  // scalar JST
        const CellState mm = load_cell(b, N, c - sd), qq = load_cell(b, N, cp + sd);
        const double fis2 = rFil * c_prm.vis2, fis4 = rFil * c_prm.vis4;
        const double ppor = (por == ADFB_NORMALFLUX) ? 0.5 : 0.0;
        const double rrad = ppor * (rad[c] + rad[cp]);
        const double dis2 = fis2 * rrad * dmin_(0.25, dmax_(dss[c], dss[cp]));
        const double dis4 = dmax_(fis4 * rrad - dis2, 0.0);
        double ddw = q.r - m.r;
        fd[0] = dis2 * ddw - dis4 * (qq.r - mm.r - 3.0 * ddw);
        ddw = q.u * q.r - m.u * m.r;
        fd[1] = dis2 * ddw - dis4 * (qq.u * qq.r - mm.u * mm.r - 3.0 * ddw);
        ddw = q.v * q.r - m.v * m.r;
        fd[2] = dis2 * ddw - dis4 * (qq.v * qq.r - mm.v * mm.r - 3.0 * ddw);
        ddw = q.w * q.r - m.w * m.r;
        fd[3] = dis2 * ddw - dis4 * (qq.w * qq.r - mm.w * mm.r - 3.0 * ddw);
        ddw = (q.e + q.p) - (m.e + m.p);
        fd[4] = dis2 * ddw - dis4 * ((qq.e + qq.p) - (mm.e + mm.p) - 3.0 * ddw);
    }
    if (DISC == ADFB_DISS_SCALAR && (APPROX & 1) && !(APPROX & 4) && doDiss) {  // inviscidDissFluxScalarApprox, blockette.F90:4367-4617
        const double ppor = (por == ADFB_NORMALFLUX) ? 0.5 : 0.0;
        const double rrad = ppor * (rad[c] + rad[cp]);
        const double dis2 = c_prm.vis2 * rrad * dmin_(0.25, dmax_(dss[c], dss[cp])) + c_prm.sigma * c_prm.vis4 * rrad;
        fd[0] = dis2 * (q.r - m.r);
        fd[1] = dis2 * (q.u * q.r - m.u * m.r);
        fd[2] = dis2 * (q.v * q.r - m.v * m.r);
        fd[3] = dis2 * (q.w * q.r - m.w * m.r);
        fd[4] = dis2 * ((q.e + q.p) - (m.e + m.p));
    }
    if (DISC == ADFB_DISS_MATRIX && doDiss) {  // matrix dissipation (exact and *Approx), blockette.F90:2515-2680
        const double gam = c_prm.gammaInf;
        const double fis2 = rFil * c_prm.vis2, fis4 = rFil * c_prm.vis4;
        const double ppor = (por == ADFB_NORMALFLUX) ? 1.0 : 0.0;
        double dr, dru, drv, drw, dre;
        if (APPROX & 5) {  // inviscidDissFluxMatrixApprox, blockette.F90:4672-4690; bit 2: ...MatrixCoarse, fluxes.F90:5205-5711
            const double dis2 = (APPROX & 4) ? rFil * c_prm.vis2Coarse * ppor
                                             : fis2 * ppor * dmin_(0.25, dmax_(dss[c], dss[cp])) + c_prm.sigma * fis4 * ppor;
            dr = dis2 * (q.r - m.r);
            dru = dis2 * (q.r * q.u - m.r * m.u);
            drv = dis2 * (q.r * q.v - m.r * m.v);
            drw = dis2 * (q.r * q.w - m.r * m.w);
            dre = dis2 * (q.e - m.e);
        } else {
            const CellState mm = load_cell(b, N, c - sd), qq = load_cell(b, N, cp + sd);
            const double dis2 = ppor * fis2 * dmin_(0.25, dmax_(dss[c], dss[cp]));
            const double dis4 = dmax_(ppor * fis4 - dis2, 0.0);
            double ddw = q.r - m.r;
            dr = dis2 * ddw - dis4 * (qq.r - mm.r - 3.0 * ddw);
            ddw = q.r * q.u - m.r * m.u;
            dru = dis2 * ddw - dis4 * (qq.r * qq.u - mm.r * mm.u - 3.0 * ddw);
            ddw = q.r * q.v - m.r * m.v;
            drv = dis2 * ddw - dis4 * (qq.r * qq.v - mm.r * mm.v - 3.0 * ddw);
            ddw = q.r * q.w - m.r * m.w;
            drw = dis2 * ddw - dis4 * (qq.r * qq.w - mm.r * mm.w - 3.0 * ddw);
            ddw = q.e - m.e;
            dre = dis2 * ddw - dis4 * (qq.e - mm.e - 3.0 * ddw);
        }
        const double gm1 = gam - 1.0, ovgm1 = 1.0 / gm1;
        const double uAvg = 0.5 * (q.u + m.u), vAvg = 0.5 * (q.v + m.v), wAvg = 0.5 * (q.w + m.w);
        const double a2Avg = 0.5 * (gam * q.p / q.r + gam * m.p / m.r);
        const double area = sqrt(s1 * s1 + s2 * s2 + s3 * s3);
        const double tmp = 1.0 / dmax_(1.e-25, area);
        const double sx = s1 * tmp, sy = s2 * tmp, sz = s3 * tmp;
        const double alphaAvg = 0.5 * (uAvg * uAvg + vAvg * vAvg + wAvg * wAvg);
        const double hAvg = alphaAvg + ovgm1 * a2Avg;
        const double aAvg = sqrt(a2Avg);
        const double unAvg = uAvg * sx + vAvg * sy + wAvg * sz;
        const double ovaAvg = 1.0 / aAvg, ova2Avg = 1.0 / a2Avg;
        double lam1 = fabs(unAvg + aAvg), lam2 = fabs(unAvg - aAvg), lam3 = fabs(unAvg);
        const double rrad = lam3 + aAvg;
        lam1 = dmax_(lam1, 0.25 * rrad) * area;
        lam2 = dmax_(lam2, 0.25 * rrad) * area;
        lam3 = dmax_(lam3, 0.025 * rrad) * area;
        const double abv1 = 0.5 * (lam1 + lam2), abv2 = 0.5 * (lam1 - lam2), abv3 = abv1 - lam3;
        const double abv4 = gm1 * (alphaAvg * dr - uAvg * dru - vAvg * drv - wAvg * drw + dre);
        const double abv5 = sx * dru + sy * drv + sz * drw - unAvg * dr;
        const double abv6 = abv3 * abv4 * ova2Avg + abv2 * abv5 * ovaAvg;
        const double abv7 = abv2 * abv4 * ovaAvg + abv3 * abv5;
        fd[0] = lam3 * dr + abv6;
        fd[1] = lam3 * dru + uAvg * abv6 + sx * abv7;
        fd[2] = lam3 * drv + vAvg * abv6 + sy * abv7;
        fd[3] = lam3 * drw + wAvg * abv6 + sz * abv7;
        fd[4] = lam3 * dre + hAvg * abv6 + unAvg * abv7;
    }
    if (DISC == ADFB_UPWIND && doDiss) {  // Roe / MUSCL, blockette.F90:3341-4363
        const CellState mm = load_cell(b, N, c - sd), qq = load_cell(b, N, cp + sd);
        const double gam = c_prm.gammaInf;
        double left[5] = {m.r, m.u, m.v, m.w, m.p}, right[5] = {q.r, q.u, q.v, q.w, q.p};
        if (!(APPROX & 1) && c_prm.limiter != ADFB_LIM_FIRSTORDER) {  // inviscidUpwindFlux(.False.) is first order
            const double du1[5] = {m.r - mm.r, m.u - mm.u, m.v - mm.v, m.w - mm.w, m.p - mm.p};
            const double du2[5] = {q.r - m.r, q.u - m.u, q.v - m.v, q.w - m.w, q.p - m.p};
            const double du3[5] = {qq.r - q.r, qq.u - q.u, qq.v - q.v, qq.w - q.w, qq.p - q.p};
            const double kappa = c_prm.kappaCoef;
            const double omk = 0.25 * (1.0 - kappa), opk = 0.25 * (1.0 + kappa);
            const double factMinmod = (3.0 - kappa) / dmax_(1.e-10, 1.0 - kappa);
#pragma unroll
            for (int l = 0; l < 5; l++) {
                double dl, dr_;
                if (c_prm.limiter == ADFB_LIM_NONE) {
                    dl = omk * du1[l] + opk * du2[l];
                    dr_ = -omk * du3[l] - opk * du2[l];
                } else {
                    const double tmp = 1.0 / copysign(dmax_(fabs(du2[l]), 1.e-10), du2[l]);
                    double rl1 = dmax_(0.0, du2[l] / copysign(dmax_(fabs(du1[l]), 1.e-10), du1[l]));
                    double rl2 = dmax_(0.0, du1[l] * tmp);
                    double rr1 = dmax_(0.0, du3[l] * tmp);
                    double rr2 = dmax_(0.0, du2[l] / copysign(dmax_(fabs(du3[l]), 1.e-10), du3[l]));
                    if (c_prm.limiter == ADFB_LIM_VANALBADA) {
                        rl1 = rl1 * (rl1 + 1.0) / (rl1 * rl1 + 1.0); rl2 = rl2 * (rl2 + 1.0) / (rl2 * rl2 + 1.0);
                        rr1 = rr1 * (rr1 + 1.0) / (rr1 * rr1 + 1.0); rr2 = rr2 * (rr2 + 1.0) / (rr2 * rr2 + 1.0);
                    } else {
                        rl1 = dmin_(1.0, factMinmod * rl1); rl2 = dmin_(1.0, factMinmod * rl2);
                        rr1 = dmin_(1.0, factMinmod * rr1); rr2 = dmin_(1.0, factMinmod * rr2);
                    }
                    dl = omk * rl1 * du1[l] + opk * rl2 * du2[l];
                    dr_ = -opk * rr1 * du2[l] - omk * rr2 * du3[l];
                }
                left[l] = dl + left[l];
                right[l] = dr_ + right[l];
            }
        }
        double porFlux = 0.5 * rFil;
        if (por == ADFB_NOFLUX || por == ADFB_BOUNDFLUX) porFlux = 0.0;
        const double gm1 = gam - 1.0, ovgm1 = 1.0 / gm1;
        const double z1l = sqrt(left[0]), z1r = sqrt(right[0]);
        double tmp = 1.0 / (z1l + z1r);
        const double Etl = left[0] * (ovgm1 * left[4] / left[0] + 0.5 * (left[1] * left[1] + left[2] * left[2] + left[3] * left[3]));
        const double Etr = right[0] * (ovgm1 * right[4] / right[0] + 0.5 * (right[1] * right[1] + right[2] * right[2] + right[3] * right[3]));
        const double dr = right[0] - left[0];
        const double dru = right[0] * right[1] - left[0] * left[1];
        const double drv = right[0] * right[2] - left[0] * left[2];
        const double drw = right[0] * right[3] - left[0] * left[3];
        const double drE = Etr - Etl;
        const double uAvg = tmp * (z1l * left[1] + z1r * right[1]);
        const double vAvg = tmp * (z1l * left[2] + z1r * right[2]);
        const double wAvg = tmp * (z1l * left[3] + z1r * right[3]);
        const double hAvg = tmp * ((Etl + left[4]) / z1l + (Etr + right[4]) / z1r);
        const double area = sqrt(s1 * s1 + s2 * s2 + s3 * s3);
        tmp = 1.0 / dmax_(1.e-25, area);
        const double sx = s1 * tmp, sy = s2 * tmp, sz = s3 * tmp;
        const double alphaAvg = 0.5 * (uAvg * uAvg + vAvg * vAvg + wAvg * wAvg);
        const double a2Avg = fabs(gm1 * (hAvg - alphaAvg));
        const double aAvg = sqrt(a2Avg);
        double unAvg = uAvg * sx + vAvg * sy + wAvg * sz;
        const double ovaAvg = 1.0 / aAvg, ova2Avg = 1.0 / a2Avg;
        if (por == ADFB_BOUNDFLUX) unAvg = 0.0;
        const double eta = 0.5 * (fabs((left[1] - right[1]) * sx + (left[2] - right[2]) * sy + (left[3] - right[3]) * sz) +
                                  fabs(sqrt(gam * left[4] / left[0]) - sqrt(gam * right[4] / right[0])));
        double lam1 = fabs(unAvg + aAvg), lam2 = fabs(unAvg - aAvg), lam3 = fabs(unAvg);
        tmp = 2.0 * eta;
        if (lam1 < tmp) lam1 = eta + 0.25 * lam1 * lam1 / eta;
        if (lam2 < tmp) lam2 = eta + 0.25 * lam2 * lam2 / eta;
        if (lam3 < tmp) lam3 = eta + 0.25 * lam3 * lam3 / eta;
        lam1 = lam1 * area; lam2 = lam2 * area; lam3 = lam3 * area;
        const double abv1 = 0.5 * (lam1 + lam2), abv2 = 0.5 * (lam1 - lam2), abv3 = abv1 - lam3;
        const double abv4 = gm1 * (alphaAvg * dr - uAvg * dru - vAvg * drv - wAvg * drw + drE);
        const double abv5 = sx * dru + sy * drv + sz * drw - unAvg * dr;
        const double abv6 = abv3 * abv4 * ova2Avg + abv2 * abv5 * ovaAvg;
        const double abv7 = abv2 * abv4 * ovaAvg + abv3 * abv5;
        // reference: flux = -porFlux*(...); fw(c) += flux; fw(cp) -= flux  ==  fd = +porFlux*(...)
        fd[0] = porFlux * (lam3 * dr + abv6);
        fd[1] = porFlux * (lam3 * dru + uAvg * abv6 + sx * abv7);
        fd[2] = porFlux * (lam3 * drv + vAvg * abv6 + sy * abv7);
        fd[3] = porFlux * (lam3 * drw + wAvg * abv6 + sz * abv7);
        fd[4] = porFlux * (lam3 * drE + hAvg * abv6 + unAvg * abv7);
    }
    if (VISCOUS && doVisc && (APPROX & 2)) {  // viscousFluxApprox (thin layer), blockette.F90:6467-6837
        double porv = 0.5 * rFil;
        if (por == ADFB_NOFLUX) porv = 0.0;
        const double* vn = b.vn + (4 * dir) * N;
        const double snrm = vn[3 * N + c];
        const double ssx = vn[c] * snrm, ssy = vn[N + c] * snrm, ssz = vn[2 * N + c] * snrm;  // d/|d|^2
        double dd = q.u - m.u;
        const double u_x = dd * ssx, u_y = dd * ssy, u_z = dd * ssz;
        dd = q.v - m.v;
        const double v_x = dd * ssx, v_y = dd * ssy, v_z = dd * ssz;
        dd = q.w - m.w;
        const double w_x = dd * ssx, w_y = dd * ssy, w_z = dd * ssz;
        dd = b.aa[cp] - b.aa[c];
        double q_x = -dd * ssx, q_y = -dd * ssy, q_z = -dd * ssz;
        const double mul = porv * (b.rlv[c] + b.rlv[cp]);
        const double mue = porv * (b.rev[c] + b.rev[cp]);
        const double mut = mul + mue;
        const double gm1 = c_prm.gammaInf - 1.0;
        const double heatCoef = mul * c_fheat[0] + mue * c_fheat[1];   // 1/(Pr gm1), 1/(Pr_t gm1)
        const double fracDiv = (2.0 * (1.0 / 3.0)) * (u_x + v_y + w_z);
        const double tauxx = mut * (2.0 * u_x - fracDiv), tauyy = mut * (2.0 * v_y - fracDiv), tauzz = mut * (2.0 * w_z - fracDiv);
        const double tauxy = mut * (u_y + v_x), tauxz = mut * (u_z + w_x), tauyz = mut * (v_z + w_y);
        q_x = heatCoef * q_x; q_y = heatCoef * q_y; q_z = heatCoef * q_z;
        const double ubar = 0.5 * (m.u + q.u), vbar = 0.5 * (m.v + q.v), wbar = 0.5 * (m.w + q.w);
        fd[1] += tauxx * s1 + tauxy * s2 + tauxz * s3;
        fd[2] += tauxy * s1 + tauyy * s2 + tauyz * s3;
        fd[3] += tauxz * s1 + tauyz * s2 + tauzz * s3;
        fd[4] += (ubar * tauxx + vbar * tauxy + wbar * tauxz) * s1 + (ubar * tauxy + vbar * tauyy + wbar * tauyz) * s2 +
                 (ubar * tauxz + vbar * tauyz + wbar * tauzz) * s3 - q_x * s1 - q_y * s2 - q_z * s3;
    }
    if (VISCOUS && doVisc && !(APPROX & 2)) {
        double porv = 0.5 * rFil;
        if (por == ADFB_NOFLUX) porv = 0.0;
        const double mul = porv * (b.rlv[c] + b.rlv[cp]);
        const double mue = porv * (b.rev[c] + b.rev[cp]);
        const double mut = mul + mue;
        const double gm1 = c_prm.gammaInf - 1.0;
        const double heatCoef = mul * c_fheat[0] + mue * c_fheat[1];   // 1/(Pr gm1), 1/(Pr_t gm1)
        const int n = c, n1 = c - t1 - t2, n2 = c - t2, n3 = c - t1;
        double g[12];
        if (GAOS) {
            const double2* p1 = reinterpret_cast<const double2*>(b.grad + (long long)n1 * 12);
            const double2* p2 = reinterpret_cast<const double2*>(b.grad + (long long)n2 * 12);
            const double2* p3 = reinterpret_cast<const double2*>(b.grad + (long long)n3 * 12);
            const double2* p0 = reinterpret_cast<const double2*>(b.grad + (long long)n * 12);
#pragma unroll
            for (int l = 0; l < 6; l++) {
                const double2 a1 = p1[l], a2 = p2[l], a3 = p3[l], a0 = p0[l];
                g[2 * l] = 0.25 * (a1.x + a2.x + a3.x + a0.x);
                g[2 * l + 1] = 0.25 * (a1.y + a2.y + a3.y + a0.y);
            }
        } else {
#pragma unroll
        for (int l = 0; l < 12; l++) {
            const double* gm = b.grad + l * N;
            g[l] = 0.25 * (gm[n1] + gm[n2] + gm[n3] + gm[n]);
        }
        }
        const double* vn = b.vn + (4 * dir) * N;
        const double ssx = vn[c], ssy = vn[N + c], ssz = vn[2 * N + c], snrm = vn[3 * N + c];
        double corr;
        corr = g[0] * ssx + g[1] * ssy + g[2] * ssz - (q.u - m.u) * snrm;
        const double u_x = g[0] - corr * ssx, u_y = g[1] - corr * ssy, u_z = g[2] - corr * ssz;
        corr = g[3] * ssx + g[4] * ssy + g[5] * ssz - (q.v - m.v) * snrm;
        const double v_x = g[3] - corr * ssx, v_y = g[4] - corr * ssy, v_z = g[5] - corr * ssz;
        corr = g[6] * ssx + g[7] * ssy + g[8] * ssz - (q.w - m.w) * snrm;
        const double w_x = g[6] - corr * ssx, w_y = g[7] - corr * ssy, w_z = g[8] - corr * ssz;
        corr = g[9] * ssx + g[10] * ssy + g[11] * ssz + (b.aa[cp] - b.aa[c]) * snrm;
        double q_x = g[9] - corr * ssx, q_y = g[10] - corr * ssy, q_z = g[11] - corr * ssz;
        const double fracDiv = (2.0 * (1.0 / 3.0)) * (u_x + v_y + w_z);
        const double tauxxS = 2.0 * u_x - fracDiv, tauyyS = 2.0 * v_y - fracDiv, tauzzS = 2.0 * w_z - fracDiv;
        const double tauxyS = u_y + v_x, tauxzS = u_z + w_x, tauyzS = v_z + w_y;
        q_x = heatCoef * q_x; q_y = heatCoef * q_y; q_z = heatCoef * q_z;
        double tauxx = mut * tauxxS, tauyy = mut * tauyyS, tauzz = mut * tauzzS;
        double tauxy = mut * tauxyS, tauxz = mut * tauxzS, tauyz = mut * tauyzS;
        if (c_prm.useQCR) {
            double den = sqrt(u_x * u_x + u_y * u_y + u_z * u_z + v_x * v_x + v_y * v_y + v_z * v_z + w_x * w_x + w_y * w_y + w_z * w_z);
            den = dmax_(den, 1.e-10);
            const double fact = mue * 0.3 / den;
            const double Wxy = u_y - v_x, Wxz = u_z - w_x, Wyz = v_z - w_y;
            const double Wyx = -Wxy, Wzx = -Wxz, Wzy = -Wyz;
            tauxx -= fact * (Wxy * tauxyS + Wxz * tauxzS) * 2.0;
            tauyy -= fact * (Wyx * tauxyS + Wyz * tauyzS) * 2.0;
            tauzz -= fact * (Wzx * tauxzS + Wzy * tauyzS) * 2.0;
            tauxy -= fact * (Wxy * tauyyS + Wxz * tauyzS + Wyx * tauxxS + Wyz * tauxzS);
            tauxz -= fact * (Wxy * tauyzS + Wxz * tauzzS + Wzx * tauxxS + Wzy * tauxyS);
            tauyz -= fact * (Wyx * tauxzS + Wyz * tauzzS + Wzx * tauxyS + Wzy * tauyyS);
        }
        const double ubar = 0.5 * (m.u + q.u), vbar = 0.5 * (m.v + q.v), wbar = 0.5 * (m.w + q.w);
        fd[1] += tauxx * s1 + tauxy * s2 + tauxz * s3;
        fd[2] += tauxy * s1 + tauyy * s2 + tauyz * s3;
        fd[3] += tauxz * s1 + tauyz * s2 + tauzz * s3;
        fd[4] += (ubar * tauxx + vbar * tauxy + wbar * tauxz) * s1 + (ubar * tauxy + vbar * tauyy + wbar * tauyz) * s2 +
                 (ubar * tauxz + vbar * tauyz + wbar * tauzz) * s3 - q_x * s1 - q_y * s2 - q_z * s3;
        if (tq) {  // storeWallTensor: viscSubface%tau, %q of a boundary face (blockette.F90:5812-5838)
            tq[0] = tauxx; tq[1] = tauyy; tq[2] = tauzz; tq[3] = tauxy; tq[4] = tauxz; tq[5] = tauyz;
            tq[6] = q_x; tq[7] = q_y; tq[8] = q_z;
        }
    }
}

// k_faces: plus faces of cell (i,j,k), i 1:il, j 1:jl, k 1:kl.  MERGED: one array G = fc - fd per
// face (net outflow of the low cell) -> flux[dir*5 + l]; otherwise fc -> flux[dir*10 + l],
// fd -> flux[dir*10 + 5 + l] (smoother path: fw persists between RK stages).
template <bool VISCOUS, bool MERGED, int DISC, int APPROX, bool STOREWALL = false, int PART = 0, bool GAOS = false>
__global__ void __launch_bounds__(FACES_TPB, PART == 0 ? FACES_MINB : FACES_MINB_SPLIT) k_faces(Dims d, BlockDev b, double rFil, int doVisc, int doDiss) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 1;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 1;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 1;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = i + sJ * j + sK * k;
    const CellState m = load_cell(b, N, c);
    double fc[5], fd[5];
    double tq[9];
    double* const tqp = STOREWALL ? tq : nullptr;
    // boundary-plane store of the wall stress tensor: plane (dir, side), in-plane index pi
    auto store_wall = [&](int dir, int side, long long pi) {
        double* dst = b.wallTau + ((long long)(dir * 2 + side) * 9) * b.wallP + pi;
#pragma unroll
        for (int l = 0; l < 9; l++) dst[l * b.wallP] = tq[l];
    };
    const bool oi = i >= 2, oj = j >= 2, ok = k >= 2;
    if (oj && ok) {
        face_flux<VISCOUS, DISC, APPROX, PART, GAOS>(b, N, c, 1, sJ, sK, 0, b.si, b.porI[c], b.radI, b.dss, m, rFil, doDiss, doVisc, fc, fd, tqp);
        if (STOREWALL && (i == 1 || i == d.il)) store_wall(0, i == 1 ? 0 : 1, j + (long long)d.NJ * k);
#pragma unroll
        for (int l = 0; l < 5; l++) {
            if (MERGED && PART == 2) b.flux[(15 + l) * N + c] = -fd[l];
            else if (MERGED) b.flux[l * N + c] = fc[l] - fd[l];
            else { b.flux[l * N + c] = fc[l]; b.flux[(5 + l) * N + c] = fd[l]; }
        }
    }
    if (oi && ok) {
        face_flux<VISCOUS, DISC, APPROX, PART, GAOS>(b, N, c, sJ, 1, sK, 1, b.sj, b.porJ[c], b.radJ, b.dss + N, m, rFil, doDiss, doVisc, fc, fd, tqp);
        if (STOREWALL && (j == 1 || j == d.jl)) store_wall(1, j == 1 ? 0 : 1, i + (long long)d.NI * k);
#pragma unroll
        for (int l = 0; l < 5; l++) {
            if (MERGED && PART == 2) b.flux[(20 + l) * N + c] = -fd[l];
            else if (MERGED) b.flux[(5 + l) * N + c] = fc[l] - fd[l];
            else { b.flux[(10 + l) * N + c] = fc[l]; b.flux[(15 + l) * N + c] = fd[l]; }
        }
    }
    if (oi && oj) {
        face_flux<VISCOUS, DISC, APPROX, PART, GAOS>(b, N, c, sK, 1, sJ, 2, b.sk, b.porK[c], b.radK, b.dss + 2 * N, m, rFil, doDiss, doVisc, fc, fd, tqp);
        if (STOREWALL && (k == 1 || k == d.kl)) store_wall(2, k == 1 ? 0 : 1, i + (long long)d.NI * j);
#pragma unroll
        for (int l = 0; l < 5; l++) {
            if (MERGED && PART == 2) b.flux[(25 + l) * N + c] = -fd[l];
            else if (MERGED) b.flux[(10 + l) * N + c] = fc[l] - fd[l];
            else { b.flux[(20 + l) * N + c] = fc[l]; b.flux[(25 + l) * N + c] = fd[l]; }
        }
    }
}

// ---------------------------------------------------------------------------
// SA residual pieces for one cell.
// saAdvection, one direction: blockette.F90:1415-1560 (k), j, i analogous
__device__ __forceinline__ double sa_adv_dir(const BlockDev& b, int N, int c, int sd, const double* __restrict__ ssum,
                                             double voli2, double ux, double uy, double uz) {
    const double* nt = b.w + ITU1 * N;
    const double xa = ssum[c] * voli2, ya = ssum[N + c] * voli2, za = ssum[2 * N + c] * voli2;
    const double uu = xa * ux + ya * uy + za * uz;
    double dwtx;
    if (uu > 0.0) {
        if (c_prm.secondOrdTurb) {
            const double dwtm1 = nt[c - sd] - nt[c - 2 * sd];
            const double dwt = nt[c] - nt[c - sd];
            const double dwtp1 = nt[c + sd] - nt[c];
            dwtx = dwt;
            if (dwt * dwtp1 > 0.0) dwtx = dwtx + 0.5 * ((fabs(dwt) < fabs(dwtp1)) ? dwt : dwtp1);
            if (dwt * dwtm1 > 0.0) dwtx = dwtx - 0.5 * ((fabs(dwt) < fabs(dwtm1)) ? dwt : dwtm1);
        } else {
            dwtx = nt[c] - nt[c - sd];
        }
    } else {
        if (c_prm.secondOrdTurb) {
            const double dwtm1 = nt[c] - nt[c - sd];
            const double dwt = nt[c + sd] - nt[c];
            const double dwtp1 = nt[c + 2 * sd] - nt[c + sd];
            dwtx = dwt;
            if (dwt * dwtp1 > 0.0) dwtx = dwtx - 0.5 * ((fabs(dwt) < fabs(dwtp1)) ? dwt : dwtp1);
            if (dwt * dwtm1 > 0.0) dwtx = dwtx + 0.5 * ((fabs(dwt) < fabs(dwtm1)) ? dwt : dwtm1);
        } else {
            dwtx = nt[c + sd] - nt[c];
        }
    }
    return uu * dwtx;
}

// saViscous, one direction: blockette.F90:1197-1258 (k), j, i analogous.
__device__ __forceinline__ double sa_visc_dir(const BlockDev& b, int N, int c, int sd, const double* __restrict__ s,
                                              const double* __restrict__ ssum, double nu, double acc) {
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
    const double xa = 0.5 * ssum[c] * voli, ya = 0.5 * ssum[N + c] * voli, za = 0.5 * ssum[2 * N + c] * voli;
    const double ttm = xm * xa + ym * ya + zm * za;
    const double ttp = xp * xa + yp * ya + zp * za;
    const double nt0 = w[ITU1 * N + c], ntm = w[ITU1 * N + cm], ntp = w[ITU1 * N + cp];
    const double cnud = -cb2 * nt0 * cb3Inv;
    const double cam = ttm * cnud, cap = ttp * cnud;
    const double nutm = 0.5 * (ntm + nt0), nutp = 0.5 * (ntp + nt0);
    const double num = 0.5 * (b.rlv[cm] / w[cm] + nu);
    const double nup = 0.5 * (b.rlv[cp] / w[cp] + nu);
    const double cdm = (num + (1.0 + cb2) * nutm) * ttm * cb3Inv;
    const double cdp = (nup + (1.0 + cb2) * nutp) * ttp * cb3Inv;
    const double c1m = dmax_(cdm + cam, 0.0), c1p = dmax_(cdp + cap, 0.0);
    const double c10 = c1m + c1p;
    return acc + c1m * ntm - c10 * nt0 + c1p * ntp;
}

// saSource: blockette.F90:976-1168
__device__ __forceinline__ double sa_source(const BlockDev& b, int N, int sJ, int sK, int c, double nu) {
    const double* w = b.w;
    double gv[3][3];
#pragma unroll
    for (int v = 0; v < 3; v++) {
        const double* q = w + (IVX + v) * N;
        const double qip = q[c + 1], qim = q[c - 1], qjp = q[c + sJ], qjm = q[c - sJ], qkp = q[c + sK], qkm = q[c - sK];
#pragma unroll
        for (int m = 0; m < 3; m++) {
            const int o = m * N;
            gv[v][m] = qip * b.si[o + c] - qim * b.si[o + c - 1] + qjp * b.sj[o + c] - qjm * b.sj[o + c - sJ] +
                       qkp * b.sk[o + c] - qkm * b.sk[o + c - sK];
        }
    }
    const double fact = 0.25 / b.vol[c];
    const double sxx = 2.0 * fact * gv[0][0], syy = 2.0 * fact * gv[1][1], szz = 2.0 * fact * gv[2][2];
    const double sxy = fact * (gv[0][1] + gv[1][0]), sxz = fact * (gv[0][2] + gv[2][0]), syz = fact * (gv[1][2] + gv[2][1]);
    const double div2 = (2.0 * (1.0 / 3.0)) * ((sxx + syy + szz) * (sxx + syy + szz));
    const double strainMag2 = 2.0 * (sxy * sxy + sxz * sxz + syz * syz) + sxx * sxx + syy * syy + szz * szz;
    double sqrtProd;
    if (c_prm.turbProd == ADFB_PROD_STRAIN) {
        sqrtProd = sqrt(dmax_(2.0 * strainMag2 - div2, 1.e-25));
    } else {
        const double vortx = 2.0 * fact * (gv[2][1] - gv[1][2]);
        const double vorty = 2.0 * fact * (gv[0][2] - gv[2][0]);
        const double vortz = 2.0 * fact * (gv[1][0] - gv[0][1]);
        sqrtProd = sqrt(vortx * vortx + vorty * vorty + vortz * vortz);
    }
    const double cv13 = c_prm.rsaCv1 * c_prm.rsaCv1 * c_prm.rsaCv1;
    const double kar2Inv = c_fheat[4];   // 1 / rsaK**2
    const double cw3 = c_prm.rsaCw3;
    const double cw36 = (cw3 * cw3 * cw3) * (cw3 * cw3 * cw3);
    const double nt = w[ITU1 * N + c];
    const double dw_ = b.d2Wall[c];
    const double dist2Inv = 1.0 / (dw_ * dw_);
    const double chi = nt / nu, chi2 = chi * chi, chi3 = chi * chi2;
    const double fv1 = chi3 / (chi3 + cv13);
    const double fv2 = 1.0 - chi / (1.0 + chi * fv1);
    double ft2 = 0.0;
    if (c_prm.useft2SA) ft2 = c_prm.rsaCt3 * exp(-c_prm.rsaCt4 * chi2);
    double sst = sqrtProd + nt * fv2 * kar2Inv * dist2Inv;
    if (c_prm.useRotationSA) sst = sst + c_prm.rsaCrot * dmin_(0.0, sqrt(2.0 * strainMag2));
    sst = dmax_(sst, 1.e-10);
    double rr = nt * kar2Inv * dist2Inv / sst;
    rr = dmin_(rr, 10.0);
    const double rr2 = rr * rr, rr6 = rr2 * rr2 * rr2;
    const double gg = rr + c_prm.rsaCw2 * (rr6 - rr);
    const double gg2 = gg * gg, gg6 = gg2 * gg2 * gg2;
    const double termFw = pow((1.0 + cw36) / (gg6 + cw36), 1.0 / 6.0);
    const double fwSa = gg * termFw;
    const double term1 = c_prm.rsaCb1 * (1.0 - ft2) * sqrtProd * (c_prm.approxSA ? 0.0 : 1.0);
    const double term2 = dist2Inv * (kar2Inv * c_prm.rsaCb1 * ((1.0 - ft2) * fv2 + ft2) - c_prm.rsaCw1 * fwSa);
    return (term1 + term2 * nt) * nt;
}

// k_sa: SA row of one owned cell: source, advection k/j/i, diffusion k/j/i, scaling
// (blockette.F90:623-627, :1872-1897)
// kOff / kTop: the owned planes 2 + kOff .. kTop only (slab pipeline); 0 / INT_MAX: all of them
__global__ void __launch_bounds__(SA_TPB, SA_MINB) k_sa(Dims d, BlockDev b, MffdEpi mf, int kOff, int kTop) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2 + kOff;
    if (i > d.il || j > d.jl || k > d.kl || k > kTop) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = i + sJ * j + sK * k;
    const double rblank = dmax_((double)b.iblank[c], 0.0);
    const double nu = b.rlv[c] / b.w[c];
    double r = 0.0;
    r = r + sa_source(b, N, sJ, sK, c, nu);
    const double voli2 = 0.5 / b.vol[c];
    const double ux = b.w[N + c], uy = b.w[2 * N + c], uz = b.w[3 * N + c];
    r = r - sa_adv_dir(b, N, c, sK, b.ssum + 6 * N, voli2, ux, uy, uz);
    r = r - sa_adv_dir(b, N, c, sJ, b.ssum + 3 * N, voli2, ux, uy, uz);
    r = r - sa_adv_dir(b, N, c, 1, b.ssum, voli2, ux, uy, uz);
    r = sa_visc_dir(b, N, c, sK, b.sk, b.ssum + 6 * N, nu, r);
    r = sa_visc_dir(b, N, c, sJ, b.sj, b.ssum + 3 * N, nu, r);
    r = sa_visc_dir(b, N, c, 1, b.si, b.ssum, nu, r);
    const double dwv = -b.volRef[c] * r * rblank;
    b.dw[ITU1 * N + c] = dwv;
    if (mf.rec) mffd_epilogue(mf, d, i, j, k, ITU1, dwv, b.volRef[c], c_prm.turbResScale);
}

// k_div: flux divergence + sumDwandFw epilogue (blockette.F90:6839-6864) for one owned cell.
// Order per variable: -Fi(c-1) +Fi(c) -Fj(c-sJ) +Fj(c) -Fk(c-sK) +Fk(c), like the reference's sweeps.
template <bool MERGED>
__global__ void __launch_bounds__(256) k_div(Dims d, BlockDev b, double rFil, int persistFw, int initWr) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = i + sJ * j + sK * k;
    const double rblank = dmax_((double)b.iblank[c], 0.0);
    const double* F = b.flux;
    if (MERGED) {
        const bool split = initWr == 2;   // k_faces ran as two launches: inviscid part in slots 0..14, viscous in 15..29
#pragma unroll
        for (int l = 0; l < 5; l++) {
            double a = 0.0;
            if (split) {
                a -= F[l * N + c - 1] + F[(15 + l) * N + c - 1];
                a += F[l * N + c] + F[(15 + l) * N + c];
                a -= F[(5 + l) * N + c - sJ] + F[(20 + l) * N + c - sJ];
                a += F[(5 + l) * N + c] + F[(20 + l) * N + c];
                a -= F[(10 + l) * N + c - sK] + F[(25 + l) * N + c - sK];
                a += F[(10 + l) * N + c] + F[(25 + l) * N + c];
            } else {
            a -= F[l * N + c - 1];
            a += F[l * N + c];
            a -= F[(5 + l) * N + c - sJ];
            a += F[(5 + l) * N + c];
            a -= F[(10 + l) * N + c - sK];
            a += F[(10 + l) * N + c];
            }
            b.dw[l * N + c] = a * rblank;
        }
    } else {
        const double sfil = 1.0 - rFil;
#pragma unroll
        for (int l = 0; l < 5; l++) {
            double a = initWr ? b.wr[l * N + c] : 0.0;   // initRes on a coarse level: dw = wr (residuals.F90:485-497)
            a -= F[l * N + c - 1];
            a += F[l * N + c];
            a -= F[(10 + l) * N + c - sJ];
            a += F[(10 + l) * N + c];
            a -= F[(20 + l) * N + c - sK];
            a += F[(20 + l) * N + c];
            double fw = persistFw ? sfil * b.fw[l * N + c] : 0.0;
            fw += F[(5 + l) * N + c - 1];
            fw -= F[(5 + l) * N + c];
            fw += F[(15 + l) * N + c - sJ];
            fw -= F[(15 + l) * N + c];
            fw += F[(25 + l) * N + c - sK];
            fw -= F[(25 + l) * N + c];
            if (persistFw) b.fw[l * N + c] = fw;
            b.dw[l * N + c] = (a + fw) * rblank;
        }
    }
}

}  // namespace

// ---------------------------------------------------------------------------
static int launch_geom(const Dims& d, const BlockDev& b, cudaStream_t stream) {
    dim3 tb(32, 4, 2);
    dim3 g((d.NI + tb.x - 1) / tb.x, (d.NJ + tb.y - 1) / tb.y, (d.NK + tb.z - 1) / tb.z);
    KT_BEGIN(K_METRICS, stream);
    k_geom<<<g, tb, 0, stream>>>(d, b);
    KT_END(K_METRICS, stream);
    return (int)cudaGetLastError();
}

// doRad: 1 = recompute spectral radii + dtl (blockette order), 0 = keep them (block/smoother path)
static bool grad_aos() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("ADFB_GRAD_AOS"); v = e ? atoi(e) : 0; }
    return v != 0;
}
static bool split_faces() {
    static int v = -1;
    if (v < 0) { const char* e = getenv("ADFB_SPLIT_FACES"); v = e ? atoi(e) : 0; }
    return v != 0;
}
// true when launch_residual_core hands the flow rows of the full exact residual in discretisation `disc` to the tile kernel
static bool tile_kernel_applies(const Dims& d, const BlockDev& b, int disc) {
    return fused_mode() > 0 && !b.coarse && disc == ADFB_DISS_SCALAR && !split_faces();
}
// disc: the discretisation of this residual (residual_discr in adflow_b200.cu); on a level above the ground level it is
// spaceDiscrCoarse and selects the first-order coarse-level fluxes
static int launch_residual_core(const Dims& d, const BlockDev& b, const AdfbParams& prm, const LaunchEnv& env, int disc, unsigned flags,
                                double rFil, int persistFw, int doRad, cudaStream_t stream, int initWr = 0, MffdEpi mf = MffdEpi{nullptr, 0}) {
    const int flowRes = (flags & ADFB_RES_FLOW) != 0;
    const int turbRes = ((flags & ADFB_RES_TURB) != 0) && prm.equations == ADFB_RANS;
    const int updateDt = 1;  // blockette timeStep always computes dtl (blockette.F90:1929-1932)
    const bool viscous = prm.equations != ADFB_EULER;
    const int doDiss = fabs(rFil) >= 1.e-10;  // fluxes.F90:1082 early return
    const int doVisc = viscous && doDiss;
    // useViscApprox only selects the thin-layer viscous flux (blockette.F90:636-644): an inviscid block ignores it
    const int dissApprox = (flags & ADFB_RES_DISS_APPROX) ? 1 : 0, viscApprox = (viscous && (flags & ADFB_RES_VISC_APPROX)) ? 1 : 0;
    if ((dissApprox || viscApprox) && persistFw) return 1;  // approximate variants exist on the blockette path only
    // experiment switch: AoS nodal-gradient store, only for the exact merged viscous scalar-JST residual (the bench path)
    const bool gradAos = grad_aos() && flowRes && doVisc && !persistFw && !dissApprox && !viscApprox && !b.coarse && !split_faces() &&
                         !((flags & ADFB_RES_STORE_WALL) != 0) && disc == ADFB_DISS_SCALAR;
    dim3 tb(32, 4, 2);
    // The SA row reads only the state and static geometry and writes dw(itu1); the flow rows write dw(1:5).
    // The two chains are independent, so k_sa is forked onto a side stream (also inside graph capture) and
    // joined at the end: both chains are latency bound, their warps interleave on the SMs.
    static int s_conc = -1;
    if (s_conc < 0) {
        const char* e = getenv("ADFB_SA_CONCURRENT");
        s_conc = e ? atoi(e) : 1;
    }
    const bool fork = turbRes && flowRes && s_conc && !g_kt.on;
    if (turbRes) {
        dim3 tr(32, 4, 1);
        dim3 g((d.nx + tr.x - 1) / tr.x, (d.ny + tr.y - 1) / tr.y, (d.nz + tr.z - 1) / tr.z);
        if (fork) {
            cudaEventRecord(env.saFork, stream);
            cudaStreamWaitEvent(env.saStream, env.saFork, 0);
            k_sa<<<g, tr, 0, env.saStream>>>(d, b, mf, 0, INT_MAX);
            g_kt.launches++; g_kt.count[K_SA]++;
            cudaEventRecord(env.saJoin, env.saStream);
        } else {
            KT_BEGIN(K_SA, stream);
            k_sa<<<g, tr, 0, stream>>>(d, b, mf, 0, INT_MAX);
            KT_END(K_SA, stream);
        }
    }
    if (doRad || (flowRes && doDiss)) {
        dim3 g((d.NI + tb.x - 1) / tb.x, (d.NJ + tb.y - 1) / tb.y, (d.NK + tb.z - 1) / tb.z);
        KT_BEGIN(K_PREP, stream);
        launch_pdl(k_prep, g, tb, stream, d, b, updateDt, doRad, 0, INT_MAX, disc, (int)!b.coarse);
        KT_END(K_PREP, stream);
    }
    // tile kernel (fused_kernels.cuh): exact central + scalar-JST (+ viscous) flow rows in one launch
    bool fusedDone = false;
    // (smoother path, persistFw: the tile kernel exchanges central and dissipative fluxes separately with two more CTA
    // barriers per plane and was slower than k_nodal/k_faces/k_div there; ADFB_FUSED_SMOOTHER=1 selects it anyway)
    static int fusedSmoother = -1;
    if (fusedSmoother < 0) { const char* e = getenv("ADFB_FUSED_SMOOTHER"); fusedSmoother = e ? atoi(e) : 0; }
    // ADFB_FUSED_SMOOTHER: 1 = the tile kernel for every smoother residual, 2 = only for the stages that form the dissipative and viscous
    // fluxes (rFil /= 0); the central-only stages keep k_faces + k_div, which are cheaper there
    if (flowRes && fused_mode() > 0 && (!persistFw || fusedSmoother == 1 || (fusedSmoother == 2 && doDiss)) && !b.coarse && disc == ADFB_DISS_SCALAR && !dissApprox && !viscApprox && !initWr &&
        !(flags & ADFB_RES_STORE_WALL) && !split_faces()) {
        KT_BEGIN(K_RESID, stream);
        const int rc = launch_flowres_tile(d, b, prm, env, (int)((b.p - b.w) / d.N), rFil, doDiss, !persistFw, persistFw, stream, mf);
        KT_END(K_RESID, stream);
        if (rc > 0) return 1;
        fusedDone = rc == 0;
    }
    if (mf.rec && flowRes && !fusedDone) return 1;   // the fused matrix-free epilogue lives in the tile kernel
    if (flowRes && doDiss && !fusedDone) {
        dim3 tn(32, 4, 2);
        dim3 g((d.ie + tn.x - 1) / tn.x, (d.je + tn.y - 1) / tn.y, (d.ke + tn.z - 1) / tn.z);
        KT_BEGIN(K_NODAL, stream);
        if (gradAos) launch_pdl(k_nodal<true>, g, tn, stream, d, b, (int)(doVisc && !viscApprox), dissApprox, disc);
        else launch_pdl(k_nodal<false>, g, tn, stream, d, b, (int)(doVisc && !viscApprox), dissApprox, disc);
        KT_END(K_NODAL, stream);
    }
    if (flowRes && !fusedDone) {
        dim3 tr(32, 4, 1);
        dim3 g((d.il + tr.x - 1) / tr.x, (d.jl + tr.y - 1) / tr.y, (d.kl + tr.z - 1) / tr.z);
        const bool merged = !persistFw;
        KT_BEGIN(K_RESID, stream);
#define ADFB_LAUNCH_FACES(V, M, D, A) launch_pdl(k_faces<V, M, D, A>, g, tr, stream, d, b, rFil, doVisc, doDiss)
#define ADFB_FACES_DISC(V, M, A)                                           \
    do {                                                                   \
        if (disc == ADFB_DISS_SCALAR) ADFB_LAUNCH_FACES(V, M, ADFB_DISS_SCALAR, A); \
        else if (disc == ADFB_DISS_MATRIX) ADFB_LAUNCH_FACES(V, M, ADFB_DISS_MATRIX, A); \
        else ADFB_LAUNCH_FACES(V, M, ADFB_UPWIND, A);                       \
    } while (0)
        const int approx = dissApprox | (viscApprox << 1);
        int splitDone = 0;
        const bool storeWall = (flags & ADFB_RES_STORE_WALL) && viscous && doVisc && merged && approx == 0;
        if (b.coarse) {   // coarse multigrid level: first-order scalar dissipation, block path only
            if (merged || approx) return 1;
            if (disc == ADFB_UPWIND) {   // inviscidUpwindFlux(fineGrid = .false.): first-order states, fluxes.F90:1532
                if (viscous) launch_pdl(k_faces<true, false, ADFB_UPWIND, 1>, g, tr, stream, d, b, rFil, doVisc, doDiss);
                else launch_pdl(k_faces<false, false, ADFB_UPWIND, 1>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            } else if (disc == ADFB_DISS_SCALAR) {
                if (viscous) launch_pdl(k_faces<true, false, ADFB_DISS_SCALAR, 4>, g, tr, stream, d, b, rFil, doVisc, doDiss);
                else launch_pdl(k_faces<false, false, ADFB_DISS_SCALAR, 4>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            } else {
                if (viscous) launch_pdl(k_faces<true, false, ADFB_DISS_MATRIX, 4>, g, tr, stream, d, b, rFil, doVisc, doDiss);
                else launch_pdl(k_faces<false, false, ADFB_DISS_MATRIX, 4>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            }
        } else if (storeWall) {  // exact viscous flux + viscSubface%tau/%q planes for the force integration
            if (disc == ADFB_DISS_SCALAR) launch_pdl(k_faces<true, true, ADFB_DISS_SCALAR, 0, true>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            else if (disc == ADFB_DISS_MATRIX) launch_pdl(k_faces<true, true, ADFB_DISS_MATRIX, 0, true>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            else launch_pdl(k_faces<true, true, ADFB_UPWIND, 0, true>, g, tr, stream, d, b, rFil, doVisc, doDiss);
        } else if (approx == 0 && viscous && merged && doVisc && split_faces()) {
            // two launches with fewer registers each (ADFB_SPLIT_FACES=1): central + dissipation, then viscous
            if (disc == ADFB_DISS_SCALAR) {
                launch_pdl(k_faces<true, true, ADFB_DISS_SCALAR, 0, false, 1>, g, tr, stream, d, b, rFil, doVisc, doDiss);
                launch_pdl(k_faces<true, true, ADFB_DISS_SCALAR, 0, false, 2>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            } else if (disc == ADFB_DISS_MATRIX) {
                launch_pdl(k_faces<true, true, ADFB_DISS_MATRIX, 0, false, 1>, g, tr, stream, d, b, rFil, doVisc, doDiss);
                launch_pdl(k_faces<true, true, ADFB_DISS_MATRIX, 0, false, 2>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            } else {
                launch_pdl(k_faces<true, true, ADFB_UPWIND, 0, false, 1>, g, tr, stream, d, b, rFil, doVisc, doDiss);
                launch_pdl(k_faces<true, true, ADFB_UPWIND, 0, false, 2>, g, tr, stream, d, b, rFil, doVisc, doDiss);
            }
            splitDone = 1;
        } else if (gradAos) {
            launch_pdl(k_faces<true, true, ADFB_DISS_SCALAR, 0, false, 0, true>, g, tr, stream, d, b, rFil, doVisc, doDiss);
        } else if (approx == 0) {
            if (viscous) { if (merged) ADFB_FACES_DISC(true, true, 0); else ADFB_FACES_DISC(true, false, 0); }
            else { if (merged) ADFB_FACES_DISC(false, true, 0); else ADFB_FACES_DISC(false, false, 0); }
        } else if (viscous) {
            if (approx == 1) ADFB_FACES_DISC(true, true, 1);
            else if (approx == 2) ADFB_FACES_DISC(true, true, 2);
            else ADFB_FACES_DISC(true, true, 3);
        } else {
            ADFB_FACES_DISC(false, true, 1);
        }
#undef ADFB_FACES_DISC
#undef ADFB_LAUNCH_FACES
        KT_END(K_RESID, stream);
        dim3 g2((d.nx + tb.x - 1) / tb.x, (d.ny + tb.y - 1) / tb.y, (d.nz + tb.z - 1) / tb.z);
        KT_BEGIN(K_DIV, stream);
        if (merged) launch_pdl(k_div<true>, g2, tb, stream, d, b, rFil, persistFw, splitDone ? 2 : 0);
        else launch_pdl(k_div<false>, g2, tb, stream, d, b, rFil, persistFw, initWr);
        KT_END(K_DIV, stream);
    }
    if (fork) cudaStreamWaitEvent(stream, env.saJoin, 0);
    return (int)cudaGetLastError();
}
