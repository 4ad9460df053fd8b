// fused_kernels.cuh -- k-marching tile kernel for the flow rows of the residual (sm_90a)
//
// One launch replaces k_nodal -> k_faces -> k_div of residual_kernels.cuh for the exact
// central + scalar-JST (+ viscous) residual, i.e. the reference's own tiled formulation
// (blocketteResCore, src/NKSolver/blockette.F90:299-753: copy a tile in, run
// inviscidCentralFlux :2150, inviscidDissFluxScalar :3029, allNodalGradients :5205,
// viscousFlux :5517 and sumDwandFw :6839 on it, write only dw) restated for a GPU:
//
//   * a CTA owns an (TX-1) x (TY-1) patch of owned cells in (i, j) plus the low-side halo
//     row/column whose threads only compute the shared faces, and marches through a chunk of
//     k planes.  Thread (ti, tj) <-> cell column (i0-1+ti, j0-1+tj).
//   * the cell state of the planes k and k+1 (rho, u, v, w, rhoE, p, rlv, rev, a^2, entropy)
//     sits in shared memory as (TX+3) x (TY+3) tiles (two halo layers for the fourth
//     differences) in a ring of three slots; the plane k+2 is in flight while plane k is
//     worked on.  The tiles arrive by TMA (cp.async.bulk.tensor, one elected thread, mbarrier
//     completion) when the leading box extent is even, else by cp.async.
//   * k direction: everything a column needs from the planes k-1 and k+2 is carried in
//     registers or read straight from global memory; the nodal gradients of node plane k-1
//     stay in registers, the sum with plane k (the k-edge sum both the i- and the j-face
//     need) and the plane-k gradients go through shared memory.
//   * each face flux is computed once (by the thread of its low-side cell), exchanged through
//     shared memory and differenced in the order the reference's sweeps touch a cell:
//     -Fi(c-1) +Fi(c) -Fj(c-sJ) +Fj(c) -Fk(c-sK) +Fk(c).  Only dw (and fw on the smoother
//     path) is written.
//
// Entropy, speed of sound squared and the spectral radii come from k_prep (one pointwise
// pass: they hold the transcendental work, which must not be redone in tile halos).
//
// The per-thread phases are plain __host__ __device__ functions of (thread context, shared
// arrays, global arrays), so that tests/emul can run the identical code thread by thread on
// the CPU (tests/test_fused_emul.py) -- test infrastructure, never a product path.
#pragma once
#include "adfb_common.cuh"
#include <math.h>

#if defined(__CUDACC__)
#define FHD __host__ __device__ __forceinline__
#else
#define FHD inline
#endif

#ifndef FT_MAXT
#define FT_MAXT 256   // max threads per CTA of the tile kernel (1 CTA / SM).  sm_90a, ptxas: 255 registers, the merged viscous kernel
                      // spills 64 B (stores) / 96 B (loads), the split one 132 / 204 B.  Two CTAs of 128 threads per SM
                      // (-DFT_MAXT=128 -DFT_S2=224 -DFT_MINB=2) get the same 255 registers and run the C2 step at 1065 against
                      // 1177 Mcells/s (one H100 SXM, 400 W limit, L2 window on)
#endif

// ring variables (shared-memory state tiles)
enum { FV_R = 0, FV_U, FV_V, FV_W, FV_E, FV_P, FV_RLV, FV_REV, FV_AA, FV_SS, FV_NUM };

// Shared-memory array sizes are compile-time constants (every offset l * FT_S0, v * FT_S2 is an immediate of the
// LDS / STS instruction); the thread tile TX x TY itself is chosen per block at run time within these bounds.
#define FT_S0 FT_MAXT   // doubles per thread-tile array (one entry per thread)
#ifndef FT_S2
#define FT_S2 352       // doubles per state tile: PX * PY <= FT_S2 (512 with FT_MAXT = 384)
#endif
#ifndef FT_MINB
#define FT_MINB 1        // resident CTAs per SM the register allocation is sized for
#endif
#ifndef FT_NSLOT
#define FT_NSLOT 3        // ring slots of the state tiles: planes k, k+1 and (3 slots) the plane k+2 in flight during step k
#endif
#define FT_NFLUX 10     // flux exchange arrays: i faces 0..4, j faces 5..9
#define FT_NFLUX_SPLIT 20   // smoother path (central and dissipative parts apart): i central 0..4, i diss 5..9, j central 10..14, j diss 15..19

struct FTile {
    int TX, TY;        // thread tile
    int PX, PY;        // state tile extents: TX+3 (rounded up to even: TMA box rows are multiples of 16 bytes), TY+3
    int nT;            // threads per CTA (TX*TY rounded up to 32)
    int kChunk;        // owned k planes per CTA
    int useTma;
    size_t smemBytes;
};

// shared-memory carve-up
struct FSmem {
    double* ring;   // [FT_NSLOT][FV_NUM][FT_S2]
    double* G;      // [FT_S0][FT_GP]  nodal gradients of node plane k (12 used)
    double* EE;     // [FT_S0][FT_GP]  k-edge sums  g(k-1) + g(k)
    double* FX;     // [FT_NFLUX][FT_S0] face fluxes
};
// nodal gradients and k-edge sums: the 12 values of a node are contiguous (pitch 14 doubles = 112 bytes: 16-byte aligned, and
// the eight lanes of a 128-bit access hit 32 distinct banks), written and read with 128-bit shared-memory accesses
#define FT_GP 14
#define FT_SMEM_DOUBLES ((size_t)FT_NSLOT * FV_NUM * FT_S2 + (size_t)(2 * FT_GP + FT_NFLUX) * FT_S0)

struct FCell { double r, u, v, w, e, p; };

struct FCtx {
    int ti, tj, i, j;
    int o2, o0;
    int c0;          // box offset of (i, j, 0)
    bool nodal;      // i <= il && j <= jl: the thread's node column exists
    bool fi, fj;     // computes the i+ / j+ faces of its cells
    bool own;        // owned cell column (writes dw)
};

struct FRegs {
    double gprev[12];   // nodal gradients of node plane k-1
    double kprev[10];   // k- face flux of the current plane (merged: 0..4; else central 0..4, dissipative 5..9)
    double qm1[5];      // conservative variables of plane k-1 (fourth difference in k)
    double dssK;        // shock sensor dss_k of plane k
    double radK;        // radK of plane k
    double svK[3];      // dual-face normal sum sv_k of layer k (the high side of node plane k-1 = the low side of node plane k)
};

// global-memory operands of one phase, loaded one phase ahead of their use (the loads of a step are in flight while the
// previous phase computes: with one CTA of <= 12 warps per SM nothing else hides their latency)
struct FGeoN { double svKhi[3], svJ[6], svI[6], ovol; };           // nodal gradients of node (i, j, k)
struct FGeoF { double s1, s2, s3, rad0, rad1, vn[4]; int por; };   // an i+ or j+ face
struct FGeoK { double s1, s2, s3, rad1, vn[4]; int por; FCell qq; double ss2; int iblank; };   // the k+ face, plane k+2 of the column

#ifndef FT_OWNCELL
#define FT_OWNCELL 0   // 1: the own cell of plane k is read once per step and kept in registers across the three faces
#endif
#ifndef FT_PAIRSUM
#define FT_PAIRSUM 1
#endif
struct FOwn { FCell m; double rlv, rev, aa, ss; };   // the thread's own cell of plane k (read once per step)

// read-only global loads through the non-coherent path
#if defined(__CUDA_ARCH__)
#define FLDG(p) __ldg(p)
// Next plane of the same operand into L2: the DRAM -> L2 transfer of step k+1's geometry overlaps the arithmetic of
// step k, so that the loads of the next step are L2 hits (no register, no scoreboard entry).
#define FPREF(p) asm volatile("prefetch.global.L2 [%0];" ::"l"(p))
#define FPREF1(p) asm volatile("prefetch.global.L1 [%0];" ::"l"(p))
#else
#define FLDG(p) (*(p))
#define FPREF(p) ((void)0)
#define FPREF1(p) ((void)0)
#endif

// ---------------------------------------------------------------------------
// flux pieces (same expressions, same order as face_flux of residual_kernels.cuh)
FHD void ff_central(const FCell& m, const FCell& q, double s1, double s2, double s3, int por, double fc[5]) {
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

FHD void ff_cons(const FCell& s, double Q[5]) {
    Q[0] = s.r; Q[1] = s.u * s.r; Q[2] = s.v * s.r; Q[3] = s.w * s.r; Q[4] = s.e + s.p;
}

// scalar JST (inviscidDissFluxScalar, blockette.F90:3133-3338); Qmm / Qqq: conservative variables of c-sd / cp+sd
FHD void ff_jst(const AdfbParams& P, const double Qmm[5], const FCell& m, const FCell& q, const double Qqq[5], int por,
                double radSum, double dssMax, double rFil, double fd[5]) {
    const double fis2 = rFil * P.vis2, fis4 = rFil * P.vis4;
    const double ppor = (por == ADFB_NORMALFLUX) ? 0.5 : 0.0;
    const double rrad = ppor * radSum;
    const double dis2 = fis2 * rrad * dmin_(0.25, dssMax);
    const double dis4 = dmax_(fis4 * rrad - dis2, 0.0);
    double ddw = q.r - m.r;
    fd[0] = dis2 * ddw - dis4 * (Qqq[0] - Qmm[0] - 3.0 * ddw);
    ddw = q.u * q.r - m.u * m.r;
    fd[1] = dis2 * ddw - dis4 * (Qqq[1] - Qmm[1] - 3.0 * ddw);
    ddw = q.v * q.r - m.v * m.r;
    fd[2] = dis2 * ddw - dis4 * (Qqq[2] - Qmm[2] - 3.0 * ddw);
    ddw = q.w * q.r - m.w * m.r;
    fd[3] = dis2 * ddw - dis4 * (Qqq[3] - Qmm[3] - 3.0 * ddw);
    ddw = (q.e + q.p) - (m.e + m.p);
    fd[4] = dis2 * ddw - dis4 * (Qqq[4] - Qmm[4] - 3.0 * ddw);
}

// viscousFlux (blockette.F90:5576-6400) of one face: g = face-averaged nodal gradients (u_x..w_z, q_x..q_z),
// vn = unit vector between the cell centres and 1/length; adds to fd[1..4]
FHD void ff_visc(const AdfbParams& P, const FCell& m, const FCell& q, double s1, double s2, double s3, int por, double rFil,
                 double rlvSum, double revSum, double daa, const double vn[4], const double g[12], double fd[5]) {
    double porv = 0.5 * rFil;
    if (por == ADFB_NOFLUX) porv = 0.0;
    const double mul = porv * rlvSum;
    const double mue = porv * revSum;
    const double mut = mul + mue;
    const double gm1 = P.gammaInf - 1.0;
#if defined(__CUDA_ARCH__)
    const double heatCoef = mul * c_fheat[0] + mue * c_fheat[1];   // the same two quotients, formed once on the host (adfb_set_params)
    (void)gm1;
#else
    const double heatCoef = mul * (1.0 / (P.prandtl * gm1)) + mue * (1.0 / (P.prandtlTurb * gm1));
#endif
    const double ssx = vn[0], ssy = vn[1], ssz = vn[2], snrm = vn[3];
    double corr;
    corr = g[0] * ssx + g[1] * ssy + g[2] * ssz - (q.u - m.u) * snrm;
    const double u_x = g[0] - corr * ssx, u_y = g[1] - corr * ssy, u_z = g[2] - corr * ssz;
    corr = g[3] * ssx + g[4] * ssy + g[5] * ssz - (q.v - m.v) * snrm;
    const double v_x = g[3] - corr * ssx, v_y = g[4] - corr * ssy, v_z = g[5] - corr * ssz;
    corr = g[6] * ssx + g[7] * ssy + g[8] * ssz - (q.w - m.w) * snrm;
    const double w_x = g[6] - corr * ssx, w_y = g[7] - corr * ssy, w_z = g[8] - corr * ssz;
    corr = g[9] * ssx + g[10] * ssy + g[11] * ssz + daa * snrm;
    double q_x = g[9] - corr * ssx, q_y = g[10] - corr * ssy, q_z = g[11] - corr * ssz;
    const double fracDiv = (2.0 * (1.0 / 3.0)) * (u_x + v_y + w_z);
    const double tauxxS = 2.0 * u_x - fracDiv, tauyyS = 2.0 * v_y - fracDiv, tauzzS = 2.0 * w_z - fracDiv;
    const double tauxyS = u_y + v_x, tauxzS = u_z + w_x, tauyzS = v_z + w_y;
    q_x = heatCoef * q_x; q_y = heatCoef * q_y; q_z = heatCoef * q_z;
    double tauxx = mut * tauxxS, tauyy = mut * tauyyS, tauzz = mut * tauzzS;
    double tauxy = mut * tauxyS, tauxz = mut * tauxzS, tauyz = mut * tauyzS;
    if (P.useQCR) {
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
}

// shock sensor of one cell and direction (blockette.F90:3091-3105)
FHD double ff_dss(double sm, double s0, double sp, double sslim) {
    return fabs((sp - 2.0 * s0 + sm) / (sp + 2.0 * s0 + sm + sslim));
}
FHD double ff_sslim_eval(const AdfbParams& P) {
    return (P.equations == ADFB_EULER) ? 0.001 * P.pInfCorr : 0.001 * P.pInfCorr / pow(P.rhoInf, P.gammaInf);
}
FHD double ff_sslim(const AdfbParams& P) {
#if defined(__CUDA_ARCH__)
    (void)P;
    return c_fheat[2];   // ff_sslim_eval(c_prm), evaluated once per parameter set on the device (k_param_consts)
#else
    return ff_sslim_eval(P);
#endif
}

FHD FCell ft_cell(const double* __restrict__ S, int o) {
    FCell s;
    s.r = S[FV_R * FT_S2 + o]; s.u = S[FV_U * FT_S2 + o]; s.v = S[FV_V * FT_S2 + o]; s.w = S[FV_W * FT_S2 + o];
    s.e = S[FV_E * FT_S2 + o]; s.p = S[FV_P * FT_S2 + o];
    return s;
}

// ---------------------------------------------------------------------------
// thread context of thread `tid` in tile (bx, by)
FHD FCtx ft_ctx(const Dims& d, const FTile& t, int tid, int bx, int by) {
    FCtx x;
    x.tj = tid / t.TX;
    x.ti = tid - x.tj * t.TX;
    x.i = 1 + bx * (t.TX - 1) + x.ti;
    x.j = 1 + by * (t.TY - 1) + x.tj;
    x.o2 = (x.tj + 1) * t.PX + (x.ti + 1);
    x.o0 = tid;
    x.c0 = x.i + (int)d.sJ * x.j;
    const bool live = x.tj < t.TY && x.i <= d.il && x.j <= d.jl;
    x.nodal = live;
    x.fi = live && x.tj >= 1;
    x.fj = live && x.ti >= 1;
    x.own = live && x.ti >= 1 && x.tj >= 1;
    return x;
}

// ---------------------------------------------------------------------------
// global-memory operand loads (issued one phase ahead of their use)
FHD void ft_load_nodal(const Dims& d, const BlockDev& b, const FCtx& x, int k, bool pf, FGeoN& g) {
    if (!x.nodal) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = x.c0 + sK * k;
    const double* __restrict__ sv = b.sv;
#pragma unroll
    for (int m = 0; m < 3; m++) {
        g.svKhi[m] = FLDG(sv + (6 + m) * N + c + sK);
        g.svJ[m] = FLDG(sv + (3 + m) * N + c);
        g.svJ[3 + m] = FLDG(sv + (3 + m) * N + c + sJ);
        g.svI[m] = FLDG(sv + m * N + c);
        g.svI[3 + m] = FLDG(sv + m * N + c + 1);
    }
    g.ovol = FLDG(b.ovol + c);
    if (pf) {
#pragma unroll
        for (int m = 0; m < 3; m++) {
            FPREF(sv + (6 + m) * N + c + 2 * sK);
            FPREF(sv + (3 + m) * N + c + sK);
            FPREF(sv + m * N + c + sK);
        }
        FPREF(b.ovol + c + sK);
    }
}
// dir 0: i+ face (s = si, rad = radI, neighbour c+1), dir 1: j+ face
FHD void ft_load_face(const Dims& d, const BlockDev& b, const FCtx& x, int k, int dir, bool visc, bool pf, FGeoF& g) {
    if (!(dir == 0 ? x.fi : x.fj)) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = x.c0 + sK * k;
    const double* __restrict__ s = dir == 0 ? b.si : b.sj;
    const double* __restrict__ rad = dir == 0 ? b.radI : b.radJ;
    g.s1 = FLDG(s + c); g.s2 = FLDG(s + N + c); g.s3 = FLDG(s + 2 * N + c);
    g.por = dir == 0 ? b.porI[c] : b.porJ[c];
    g.rad0 = FLDG(rad + c);
    g.rad1 = FLDG(rad + c + (dir == 0 ? 1 : sJ));
    if (visc) {
#pragma unroll
        for (int l = 0; l < 4; l++) g.vn[l] = FLDG(b.vn + (4 * dir + l) * N + c);
    }
    if (pf) {
        FPREF(s + c + sK); FPREF(s + N + c + sK); FPREF(s + 2 * N + c + sK);
        FPREF(rad + c + sK);
        if (visc) {
#pragma unroll
            for (int l = 0; l < 4; l++) FPREF(b.vn + (4 * dir + l) * N + c + sK);
        }
    }
}
FHD void ft_load_face_k(const Dims& d, const BlockDev& b, const FCtx& x, int k, bool visc, int doDiss, bool pf, FGeoK& g) {
    if (!x.own) return;
    const int N = (int)d.N, sK = (int)d.sK;
    const int c = x.c0 + sK * k;
    g.s1 = FLDG(b.sk + c); g.s2 = FLDG(b.sk + N + c); g.s3 = FLDG(b.sk + 2 * N + c);
    g.por = b.porK[c];
    g.rad1 = FLDG(b.radK + c + sK);
    g.iblank = b.iblank[c];
    if (visc) {
#pragma unroll
        for (int l = 0; l < 4; l++) g.vn[l] = FLDG(b.vn + (8 + l) * N + c);
    }
    if (doDiss) {   // plane k+2 of the own column straight from global memory
        const int c2 = c + 2 * sK;
        g.qq.r = FLDG(b.w + c2); g.qq.u = FLDG(b.w + N + c2); g.qq.v = FLDG(b.w + 2 * N + c2); g.qq.w = FLDG(b.w + 3 * N + c2);
        g.qq.e = FLDG(b.w + 4 * N + c2); g.qq.p = FLDG(b.p + c2);
        g.ss2 = FLDG(b.ss + c2);
    }
    if (pf) {
        FPREF(b.sk + c + sK); FPREF(b.sk + N + c + sK); FPREF(b.sk + 2 * N + c + sK);
        FPREF(b.radK + c + 2 * sK);
        if (visc) {
#pragma unroll
            for (int l = 0; l < 4; l++) FPREF(b.vn + (8 + l) * N + c + sK);
        }
    }
}

// FT_PFL1 = 1: at the start of a step every thread asks for the face operands of THIS step in L1 (they are read one to
// three phases later); pays only when shared memory leaves L1 room for them (FT_MAXT <= 256: ~100 KB of L1)
#ifndef FT_PFL1
#define FT_PFL1 0
#endif
FHD void ft_prefetch_faces_l1(const Dims& d, const BlockDev& b, const FCtx& x, int k, bool visc, int doDiss, bool doIJ) {
    if (!(x.fi || x.fj)) return;
    const int N = (int)d.N, sJ = (int)d.sJ, sK = (int)d.sK;
    const int c = x.c0 + sK * k;
    (void)N; (void)sJ; (void)c;
    if (doIJ) {
#pragma unroll
        for (int m = 0; m < 3; m++) { FPREF1(b.si + m * N + c); FPREF1(b.sj + m * N + c); }
        FPREF1(b.radI + c); FPREF1(b.radJ + c); FPREF1(b.radJ + c + sJ);
        if (visc) {
#pragma unroll
            for (int l = 0; l < 8; l++) FPREF1(b.vn + l * N + c);
        }
    }
    if (x.own) {
#pragma unroll
        for (int m = 0; m < 3; m++) FPREF1(b.sk + m * N + c);
        FPREF1(b.radK + c + sK);
        if (visc) {
#pragma unroll
            for (int l = 8; l < 12; l++) FPREF1(b.vn + l * N + c);
        }
        if (doDiss) {
            const int c2 = c + 2 * sK;
#pragma unroll
            for (int l = 0; l < 5; l++) FPREF1(b.w + l * N + c2);
            FPREF1(b.p + c2); FPREF1(b.ss + c2);
        }
    }
}

// ---------------------------------------------------------------------------
// phase 1: nodal gradients of node (i, j, k) (allNodalGradients, blockette.F90:5205-5515, gather form as k_nodal)
// from the planes k (A) and k+1 (B); stores g(k) and, when withE, the k-edge sum g(k-1)+g(k); g(k) becomes gprev.
FHD void ft_nodal(const FTile& t, const FCtx& x, const double* __restrict__ A, const double* __restrict__ B, const FGeoN& gn, FSmem& sm,
                  FRegs& r, bool withE) {
    if (!x.nodal) return;
    const int PX = t.PX;
    double q[8][4];
#pragma unroll
    for (int m = 0; m < 8; m++) {
        const double* S = (m & 4) ? B : A;
        const int o = x.o2 + (m & 1) + ((m >> 1) & 1) * PX;
        q[m][0] = S[FV_U * FT_S2 + o]; q[m][1] = S[FV_V * FT_S2 + o]; q[m][2] = S[FV_W * FT_S2 + o]; q[m][3] = S[FV_AA * FT_S2 + o];
    }
    double bar[6][4];   // [K lo, K hi, J lo, J hi, I lo, I hi]
#if FT_PAIRSUM
    // the six dual-face averages of each variable from shared pair sums (14 additions instead of 18; the
    // reference adds the four cells left to right, the difference is one rounding)
#pragma unroll
    for (int v = 0; v < 4; v++) {
        const double p01 = q[0][v] + q[1][v], p23 = q[2][v] + q[3][v], p45 = q[4][v] + q[5][v], p67 = q[6][v] + q[7][v];
        const double p02 = q[0][v] + q[2][v], p13 = q[1][v] + q[3][v], p46 = q[4][v] + q[6][v], p57 = q[5][v] + q[7][v];
        bar[0][v] = 0.25 * (p01 + p23); bar[1][v] = 0.25 * (p45 + p67);
        bar[2][v] = 0.25 * (p01 + p45); bar[3][v] = 0.25 * (p23 + p67);
        bar[4][v] = 0.25 * (p02 + p46); bar[5][v] = 0.25 * (p13 + p57);
    }
#else
    {
        const int lo[3][4] = {{0, 2, 4, 6}, {0, 1, 4, 5}, {0, 1, 2, 3}};
        const int hi[3][4] = {{1, 3, 5, 7}, {2, 3, 6, 7}, {4, 5, 6, 7}};
#pragma unroll
        for (int dd = 0; dd < 3; dd++)
#pragma unroll
            for (int side = 0; side < 2; side++) {
                const int* sel = side ? hi[dd] : lo[dd];
#pragma unroll
                for (int v = 0; v < 4; v++) bar[2 * (2 - dd) + side][v] = 0.25 * (q[sel[0]][v] + q[sel[1]][v] + q[sel[2]][v] + q[sel[3]][v]);
            }
    }
#endif
    double g[12];
#pragma unroll
    for (int m = 0; m < 12; m++) g[m] = 0.0;
#pragma unroll
    for (int dd = 2; dd >= 0; dd--) {  // K, J, I
#pragma unroll
        for (int side = 0; side < 2; side++) {
            const double* sv = dd == 2 ? (side ? gn.svKhi : r.svK) : dd == 1 ? gn.svJ + 3 * side : gn.svI + 3 * side;
            const double s1 = sv[0], s2 = sv[1], s3 = sv[2];
            const double* br = bar[2 * (2 - dd) + side];
            const double sg = side ? 1.0 : -1.0;
#pragma unroll
            for (int v = 0; v < 3; v++) {
                g[3 * v + 0] += sg * (br[v] * s1);
                g[3 * v + 1] += sg * (br[v] * s2);
                g[3 * v + 2] += sg * (br[v] * s3);
            }
            g[9] -= sg * (br[3] * s1);
            g[10] -= sg * (br[3] * s2);
            g[11] -= sg * (br[3] * s3);
        }
    }
#pragma unroll
    for (int m = 0; m < 3; m++) r.svK[m] = gn.svKhi[m];
    const double oVol = gn.ovol;
    double2* Gd = reinterpret_cast<double2*>(sm.G + (size_t)x.o0 * FT_GP);
    double2* Ed = reinterpret_cast<double2*>(sm.EE + (size_t)x.o0 * FT_GP);
#pragma unroll
    for (int m = 0; m < 6; m++) {
        const double g0 = g[2 * m] * oVol, g1 = g[2 * m + 1] * oVol;
        Gd[m] = make_double2(g0, g1);
        if (withE) Ed[m] = make_double2(r.gprev[2 * m] + g0, r.gprev[2 * m + 1] + g1);
        r.gprev[2 * m] = g0; r.gprev[2 * m + 1] = g1;
    }
}

// phase 2a: the i+ (dir 0) or j+ (dir 1) face of cell (i, j, k): fc (central) and fd (JST + viscous)
template <bool VISCOUS>
FHD void ft_face_ij(const AdfbParams& P, const FTile& t, const FCtx& x, int dir, const double* __restrict__ A, const FSmem& sm, const FGeoF& gf,
                    const FOwn& ow, double rFil, int doDiss, double fc[5], double fd[5]) {
    const int so = dir == 0 ? 1 : t.PX;        // state-tile offset of the neighbour across the face
    const int eo = dir == 0 ? t.TX : 1;        // thread-tile offset of the second node column of the face (i face: j-1, j face: i-1)
    const int o = x.o2;
#if FT_OWNCELL
    const FCell& m = ow.m;
#else
    const FCell m = ft_cell(A, o);
#endif
    const FCell q = ft_cell(A, o + so);
    ff_central(m, q, gf.s1, gf.s2, gf.s3, gf.por, fc);
#pragma unroll
    for (int l = 0; l < 5; l++) fd[l] = 0.0;
    if (doDiss) {
        const FCell mm = ft_cell(A, o - so), qq = ft_cell(A, o + 2 * so);
        double Qmm[5], Qqq[5];
        ff_cons(mm, Qmm); ff_cons(qq, Qqq);
        const double* ss = A + FV_SS * FT_S2;
        const double sslim = ff_sslim(P);
        const double ssp = ss[o + so];
        const double ss0 = FT_OWNCELL ? ow.ss : ss[o];
        const double d0 = ff_dss(ss[o - so], ss0, ssp, sslim), d1 = ff_dss(ss0, ssp, ss[o + 2 * so], sslim);
        ff_jst(P, Qmm, m, q, Qqq, gf.por, gf.rad0 + gf.rad1, dmax_(d0, d1), rFil, fd);
    }
    if (VISCOUS && doDiss) {
        double g[12];
#pragma unroll
        {
            const double2* Ea = reinterpret_cast<const double2*>(sm.EE + (size_t)(x.o0 - eo) * FT_GP);
            const double2* Eb = reinterpret_cast<const double2*>(sm.EE + (size_t)x.o0 * FT_GP);
#pragma unroll
            for (int l = 0; l < 6; l++) {
                const double2 a = Ea[l], c = Eb[l];
                g[2 * l] = 0.25 * (a.x + c.x); g[2 * l + 1] = 0.25 * (a.y + c.y);
            }
        }
        ff_visc(P, m, q, gf.s1, gf.s2, gf.s3, gf.por, rFil, (FT_OWNCELL ? ow.rlv : A[FV_RLV * FT_S2 + o]) + A[FV_RLV * FT_S2 + o + so],
                (FT_OWNCELL ? ow.rev : A[FV_REV * FT_S2 + o]) + A[FV_REV * FT_S2 + o + so],
                A[FV_AA * FT_S2 + o + so] - (FT_OWNCELL ? ow.aa : A[FV_AA * FT_S2 + o]), gf.vn, g, fd);
    }
}

// phase 2b: the k+ face of the own column (planes k | k+1); updates the carried k-direction registers
template <bool VISCOUS>
FHD void ft_face_k(const AdfbParams& P, const FTile& t, const FCtx& x, const double* __restrict__ A, const double* __restrict__ B, const FSmem& sm,
                   const FGeoK& gk, const FOwn& ow, FRegs& r, double rFil, int doDiss, double fc[5], double fd[5]) {
    const int o = x.o2, TX = t.TX;
#if FT_OWNCELL
    const FCell& m = ow.m;
#else
    const FCell m = ft_cell(A, o);
#endif
    const FCell q = ft_cell(B, o);
    ff_central(m, q, gk.s1, gk.s2, gk.s3, gk.por, fc);
#pragma unroll
    for (int l = 0; l < 5; l++) fd[l] = 0.0;
    if (doDiss) {
        double Qqq[5];
        ff_cons(gk.qq, Qqq);
        const double d1 = ff_dss(FT_OWNCELL ? ow.ss : A[FV_SS * FT_S2 + o], B[FV_SS * FT_S2 + o], gk.ss2, ff_sslim(P));
        ff_jst(P, r.qm1, m, q, Qqq, gk.por, r.radK + gk.rad1, dmax_(r.dssK, d1), rFil, fd);
        r.dssK = d1;
    }
    r.radK = gk.rad1;
    if (VISCOUS && doDiss) {
        double g[12];
        {
            const double2* G1 = reinterpret_cast<const double2*>(sm.G + (size_t)(x.o0 - TX - 1) * FT_GP);
            const double2* G2 = reinterpret_cast<const double2*>(sm.G + (size_t)(x.o0 - TX) * FT_GP);
            const double2* G3 = reinterpret_cast<const double2*>(sm.G + (size_t)(x.o0 - 1) * FT_GP);
#pragma unroll
            for (int l = 0; l < 6; l++) {   // own node: still in registers
                const double2 a = G1[l], c = G2[l], e = G3[l];
                g[2 * l] = 0.25 * (a.x + c.x + e.x + r.gprev[2 * l]); g[2 * l + 1] = 0.25 * (a.y + c.y + e.y + r.gprev[2 * l + 1]);
            }
        }
        ff_visc(P, m, q, gk.s1, gk.s2, gk.s3, gk.por, rFil, (FT_OWNCELL ? ow.rlv : A[FV_RLV * FT_S2 + o]) + B[FV_RLV * FT_S2 + o],
                (FT_OWNCELL ? ow.rev : A[FV_REV * FT_S2 + o]) + B[FV_REV * FT_S2 + o], B[FV_AA * FT_S2 + o] - (FT_OWNCELL ? ow.aa : A[FV_AA * FT_S2 + o]),
                gk.vn, g, fd);
    }
    ff_cons(m, r.qm1);
}

// what the first (prologue) step of a chunk needs from below: conservative variables and sensor of plane k-1, sv_k of layer k
FHD void ft_prologue_regs(const AdfbParams& P, const Dims& d, const BlockDev& b, const FCtx& x, int k, FRegs& r, int doDiss, bool visc) {
#pragma unroll
    for (int l = 0; l < 12; l++) r.gprev[l] = 0.0;
#pragma unroll
    for (int l = 0; l < 10; l++) r.kprev[l] = 0.0;
#pragma unroll
    for (int l = 0; l < 5; l++) r.qm1[l] = 0.0;
    r.dssK = 0.0; r.radK = 0.0;
    r.svK[0] = r.svK[1] = r.svK[2] = 0.0;
    const int N = (int)d.N, sK = (int)d.sK;
    const int c = x.c0 + sK * k, cm = c - sK;
    if (x.nodal && visc && doDiss) {
#pragma unroll
        for (int m = 0; m < 3; m++) r.svK[m] = FLDG(b.sv + (6 + m) * N + c);
    }
    if (!x.own) return;
    r.radK = FLDG(b.radK + c);
    if (!doDiss) return;
    FCell mm;
    mm.r = FLDG(b.w + cm); mm.u = FLDG(b.w + N + cm); mm.v = FLDG(b.w + 2 * N + cm); mm.w = FLDG(b.w + 3 * N + cm);
    mm.e = FLDG(b.w + 4 * N + cm); mm.p = FLDG(b.p + cm);
    ff_cons(mm, r.qm1);
    r.dssK = ff_dss(FLDG(b.ss + cm), FLDG(b.ss + c), FLDG(b.ss + c + sK), ff_sslim(P));
}

// One k step of one thread, cut at the two CTA-wide synchronisation points of the merged path (A | B) and at the two
// extra ones of the smoother path, where central and dissipative fluxes are exchanged separately and the i and j
// exchanges share the flux arrays (B1, B2):
//   ft_step_a : nodal gradients of node plane k                                           -> G, EE
//   ft_step_b : i+, j+ (merged: both) and k+ faces                                         -> FX, kp
//   ft_step_c : flux divergence in the reference's order + sumDwandFw epilogue (as k_div)  -> dw (fw)
struct FStep {
    FGeoN gn;     // operands of the NEXT nodal phase (loaded during ft_step_b)
    FGeoF gi, gj;
    FGeoK gk;
    double kp[10];
};

template <bool MERGED>
FHD void ft_store_flux(const FCtx& x, FSmem& sm, int slot, const double fc[5], const double fd[5]) {
#pragma unroll
    for (int l = 0; l < 5; l++) {
        if (MERGED) sm.FX[(slot + l) * FT_S0 + x.o0] = fc[l] - fd[l];
        else { sm.FX[(2 * slot + l) * FT_S0 + x.o0] = fc[l]; sm.FX[(2 * slot + 5 + l) * FT_S0 + x.o0] = fd[l]; }
    }
}

// divergence of cell (i, j, k): -Fi(c-1) +Fi(c) -Fj(c-sJ) +Fj(c) -Fk(c-sK) +Fk(c) per variable, then the epilogue
template <bool MERGED>
FHD void ft_div(const Dims& d, const BlockDev& b, const FTile& t, const FCtx& x, int k, const FSmem& sm, FRegs& r, FStep& st, double rFil,
                int persistFw, const MffdEpi& mf, double turbScale) {
    if (!x.own) return;
    const int N = (int)d.N, sK = (int)d.sK, TX = t.TX;
    const int c = x.c0 + sK * k;
    const double rblank = dmax_((double)st.gk.iblank, 0.0);
    const double* F = sm.FX;
    const int q0 = x.o0;
    if (MERGED) {
#pragma unroll
        for (int l = 0; l < 5; l++) {
            double a = 0.0;
            a -= F[l * FT_S0 + q0 - 1];
            a += F[l * FT_S0 + q0];
            a -= F[(5 + l) * FT_S0 + q0 - TX];
            a += F[(5 + l) * FT_S0 + q0];
            a -= r.kprev[l];
            a += st.kp[l];
            const double dwv = a * rblank;
            b.dw[l * N + c] = dwv;
            if (mf.rec) mffd_epilogue(mf, d, x.i, x.j, k, l, dwv, b.volRef[c], turbScale);
        }
    } else {   // smoother path: central part -> dw, dissipative + viscous part blended into the persistent fw
        const double sfil = 1.0 - rFil;
#pragma unroll
        for (int l = 0; l < 5; l++) {
            double a = 0.0;
            a -= F[l * FT_S0 + q0 - 1];
            a += F[l * FT_S0 + q0];
            a -= F[(10 + l) * FT_S0 + q0 - TX];
            a += F[(10 + l) * FT_S0 + q0];
            a -= r.kprev[l];
            a += st.kp[l];
            double fw = persistFw ? sfil * b.fw[l * N + c] : 0.0;
            fw += F[(5 + l) * FT_S0 + q0 - 1];
            fw -= F[(5 + l) * FT_S0 + q0];
            fw += F[(15 + l) * FT_S0 + q0 - TX];
            fw -= F[(15 + l) * FT_S0 + q0];
            fw += r.kprev[5 + l];
            fw -= st.kp[5 + l];
            if (persistFw) b.fw[l * N + c] = fw;
            b.dw[l * N + c] = (a + fw) * rblank;
        }
    }
}
// global source of ring variable v
FHD const double* ft_var_ptr(const Dims& d, const BlockDev& b, int v) {
    switch (v) {
        case FV_P: return b.p;
        case FV_RLV: return b.rlv;
        case FV_REV: return b.rev;
        case FV_AA: return b.aa;
        case FV_SS: return b.ss;
        default: return b.w + (long long)v * d.N;
    }
}
FHD bool ft_var_used(int v, bool viscous, int doDiss) {
    // laminar runs read the (zero) eddy viscosity like the general kernels do
    if (v == FV_RLV || v == FV_REV || v == FV_AA) return viscous && doDiss;
    if (v == FV_SS) return doDiss != 0;
    return true;
}

// The step driver shared by the kernel and the CPU emulation: SYNC is the CTA barrier (a no-op functor on the CPU, where
// the caller runs every thread up to each cut instead).  Kept as three plain functions so that both drivers call the
// same per-thread code between the same synchronisation points.
// FT_EARLY = 1: the global operands of a phase are loaded one phase ahead of their use (needs the registers: FT_MAXT <=
// 256); 0: right before their use (the L2 prefetch of the previous step covers part of the latency)
#ifndef FT_EARLY
#define FT_EARLY 0
#endif
// FT_AHEAD (bits): 1 / 2 = the operands of the j / k face are requested before the i face is formed (their L2 latency hides
// behind its arithmetic); 4 = the nodal operands of the next plane at the end of the step; 8 = the i-face operands before the
// barrier that follows the nodal phase.  On sm_90a every setting runs at the 255-register cap and the requests ahead cost spills
// (merged kernel, ptxas: 0 -> 64 B, 1 -> 100 B, 2 -> 96 B, 3 -> 140 B of spill stores).  C2 on one H100 SXM (400 W limit), tile
// kernel / residual step: 0 -> 154 us / 1396 Mcells/s, 1 -> 165 / 1358, 2 -> 171 / 1370, 3 -> 172 / 1317; default 0
#ifndef FT_AHEAD
#define FT_AHEAD 0
#endif
template <bool VISCOUS, bool MERGED>
FHD void ft_step_a(const Dims& d, const BlockDev& b, const FTile& t, const FCtx& x, int k, int kb, const double* A, const double* B, FSmem& sm,
                   FRegs& r, FStep& st, int doDiss, bool doIJ) {
    const bool visc = VISCOUS && doDiss;
    const bool pf = k < kb;
    if (FT_PFL1) ft_prefetch_faces_l1(d, b, x, k, visc, doDiss, doIJ);
    if (FT_EARLY) {
        // face operands of this step: in flight during the nodal phase (gn was loaded during the previous step's k face)
        if (doIJ) { ft_load_face(d, b, x, k, 0, visc, pf, st.gi); ft_load_face(d, b, x, k, 1, visc, pf, st.gj); }
        ft_load_face_k(d, b, x, k, visc, doDiss, pf, st.gk);
        if (visc) ft_nodal(t, x, A, B, st.gn, sm, r, doIJ);
    } else if (visc) {
        if (!(FT_AHEAD & (4 | 16))) ft_load_nodal(d, b, x, k, pf, st.gn);   // bits 4 / 16: requested during the previous step (and in the prologue)
        ft_nodal(t, x, A, B, st.gn, sm, r, doIJ);
    }
    // bit 8: the i-face operands are requested here, before the barrier that follows the nodal phase
    if (!FT_EARLY && (FT_AHEAD & 8) && doIJ && x.fi) ft_load_face(d, b, x, k, 0, visc, pf, st.gi);
}
// i, j and k faces between the two barriers (`part` is kept for experiments: 0 = i face only, 1 = j + k faces only, 2 = all)
template <bool VISCOUS, bool MERGED>
FHD void ft_step_b(const AdfbParams& P, const Dims& d, const BlockDev& b, const FTile& t, const FCtx& x, int k, int kb, const double* A,
                   const double* B, FSmem& sm, FRegs& r, FStep& st, double rFil, int doDiss, bool doIJ, int part) {
    const bool visc = VISCOUS && doDiss;
    const bool pf = k < kb;
    double fc[5], fd[5];
    FOwn ow;
    if (FT_OWNCELL && (x.fi || x.fj)) {
        ow.m = ft_cell(A, x.o2);
        ow.ss = doDiss ? A[FV_SS * FT_S2 + x.o2] : 0.0;
        ow.rlv = visc ? A[FV_RLV * FT_S2 + x.o2] : 0.0;
        ow.rev = visc ? A[FV_REV * FT_S2 + x.o2] : 0.0;
        ow.aa = visc ? A[FV_AA * FT_S2 + x.o2] : 0.0;
    }
    // FT_AHEAD bits 1 / 2: the face operands of the j and k faces are requested BEFORE the i face is formed
    if (!FT_EARLY && part == 2) {
        if ((FT_AHEAD & 1) && doIJ && x.fj) ft_load_face(d, b, x, k, 1, visc, pf, st.gj);
        if ((FT_AHEAD & 2) && x.own) ft_load_face_k(d, b, x, k, visc, doDiss, pf, st.gk);
    }
    if (part != 1) {
        if (FT_EARLY && visc && k < kb) ft_load_nodal(d, b, x, k + 1, k + 1 < kb, st.gn);   // for the next step's nodal phase
        if (doIJ && x.fi) {
            if (!FT_EARLY && !(FT_AHEAD & 8)) ft_load_face(d, b, x, k, 0, visc, pf, st.gi);
            ft_face_ij<VISCOUS>(P, t, x, 0, A, sm, st.gi, ow, rFil, doDiss, fc, fd);
            ft_store_flux<MERGED>(x, sm, 0, fc, fd);
        }
    }
    if (part != 0) {
        if (doIJ && x.fj) {
            if (!FT_EARLY && !((FT_AHEAD & 1) && part == 2)) ft_load_face(d, b, x, k, 1, visc, pf, st.gj);
            ft_face_ij<VISCOUS>(P, t, x, 1, A, sm, st.gj, ow, rFil, doDiss, fc, fd);
            ft_store_flux<MERGED>(x, sm, 5, fc, fd);
        }
        if (x.own) {
            if (!FT_EARLY && !((FT_AHEAD & 2) && part == 2)) ft_load_face_k(d, b, x, k, visc, doDiss, pf, st.gk);
            ft_face_k<VISCOUS>(P, t, x, A, B, sm, st.gk, ow, r, rFil, doDiss, fc, fd);
#pragma unroll
            for (int l = 0; l < 5; l++) {
                if (MERGED) st.kp[l] = fc[l] - fd[l];
                else { st.kp[l] = fc[l]; st.kp[5 + l] = fd[l]; }
            }
        }
    }
    if (!FT_EARLY && (FT_AHEAD & 4) && visc && k < kb && part != 0) ft_load_nodal(d, b, x, k + 1, k + 1 < kb, st.gn);
}

// ---------------------------------------------------------------------------
// tile selection (host)
static inline FTile ftile_make(int TX, int TY, int kChunk, bool tma) {
    FTile t;
    t.TX = TX; t.TY = TY; t.PX = (TX + 3 + 1) & ~1; t.PY = TY + 3;
    t.nT = ((TX * TY + 31) / 32) * 32;
    t.kChunk = kChunk;
    t.useTma = tma ? 1 : 0;
    t.smemBytes = FT_SMEM_DOUBLES * sizeof(double) + 64 /* mbarriers */;
    return t;
}
static inline bool ftile_fits(const FTile& t) { return t.nT <= FT_MAXT && t.PX * t.PY <= FT_S2 && t.TX >= 2 && t.TY >= 2; }

// Pick the thread tile for a block: (TX-1) x (TY-1) owned cells per CTA within the compile-time array sizes; score =
// owned cells per thread slot, with a preference for more threads per SM; the k chunk is sized so that the grid is
// close to a whole number of waves of one CTA per SM.
static inline FTile ftile_choose(const Dims& d, bool tma, int nSM) {
    int ox = 0, oy = 0, okc = 0;
    if (const char* e = getenv("ADFB_TILE")) sscanf(e, "%d,%d,%d", &ox, &oy, &okc);
    // One CTA per SM, and the time of a k plane grows with the warps of the CTA (the kernel is issue bound inside the CTA): modelled
    // as 2.3 + 0.69 x warps per plane (relative units).  The cost of a choice is waves x (planes per chunk + the prologue step, ~0.45
    // of a plane) x that time.  The SM count is the device's, so the pick follows the part: on one H100 SXM (132 SMs, 400 W limit)
    // the C2 residual step runs at 1401 Mcells/s with the pick, against 1072-1260 with fixed ADFB_TILE choices (17,13,16 13,19,5
    // 15,15,8 11,17,8 19,11,16).
    FTile best = ftile_make(tma ? 9 : 8, 4, d.nz, tma);
    double bestCost = 1e300;
    for (int pass = 0; pass < 2 && bestCost >= 1e300; pass++) {   // pass 0 honours ADFB_TILE, pass 1 (override does not fit) searches freely
        for (int TX = 4; TX <= 128; TX++) {
            for (int TY = 3; TY <= 64; TY++) {
                if (pass == 0 && ox > 0 && (TX != ox || TY != oy)) continue;
                FTile t = ftile_make(TX, TY, d.nz, tma);
                if (!ftile_fits(t) || (tma && !(TX & 1))) continue;   // TMA: the tile origin bx*(TX-1) must be 16-byte aligned
                const int nti = (d.nx + TX - 2) / (TX - 1), ntj = (d.ny + TY - 2) / (TY - 1);
                const long long cols = (long long)nti * ntj;
                // rows that are whole half-warps keep the 64-bit shared-memory accesses conflict free
                const double bank = (TX % 16 == 0) ? 1.0 : 0.93;
                for (int n = 1; n <= d.nz; n++) {
                    int kc = (d.nz + n - 1) / n;
                    if (pass == 0 && okc > 0) kc = okc;
                    if (kc < 2 && n > 1) break;
                    const long long ctas = cols * ((d.nz + kc - 1) / kc);
                    const long long waves = (ctas + nSM - 1) / nSM;
                    const double cost = (double)waves * (kc + 0.45) * (2.3 + 0.69 * (t.nT / 32)) / bank;
                    if (cost < bestCost - 1e-9) { bestCost = cost; best = t; best.kChunk = kc; }
                    if (pass == 0 && okc > 0) break;
                }
            }
        }
    }
    return best;
}

// ===========================================================================
// device side
#if defined(__CUDACC__)
#include <cuda.h>   // CUtensorMap (types only; the encoder is fetched through cudaGetDriverEntryPoint)

namespace {

__device__ __forceinline__ unsigned ft_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void ft_cp_async8(double* dst, const double* src, bool valid) {
    const unsigned n = valid ? 8u : 0u;   // src-size 0: the 8 bytes are zero-filled, nothing is read
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8, %2;\n" ::"r"(ft_smem_u32(dst)), "l"(src), "r"(n) : "memory");
}
__device__ __forceinline__ void ft_cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void ft_cp_async_wait_all() { asm volatile("cp.async.wait_group 0;\n" ::: "memory"); }

__device__ __forceinline__ void ft_mbar_init(unsigned long long* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(ft_smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void ft_mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(ft_smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void ft_mbar_wait(unsigned long long* bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(ft_smem_u32(bar)), "r"(parity) : "memory");
}
// one (PX, PY, 1) box of a (NI, NJ, NK*ncomp) tensor -> shared memory, completion on an mbarrier
__device__ __forceinline__ void ft_tma_load_3d(double* dst, const CUtensorMap* map, int x, int y, int z, unsigned long long* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(ft_smem_u32(dst)),
                 "l"(map), "r"(x), "r"(y), "r"(z), "r"(ft_smem_u32(bar))
                 : "memory");
}

struct FTmaMaps { CUtensorMap slab, aa, ss; };

// Flow rows of the residual for one (i, j) tile and one chunk of k planes.
extern __shared__ __align__(128) double ft_smem[];

#ifndef FT_LB
#define FT_LB FT_MAXT   // launch bound: FT_LB > FT_MAXT caps the registers below 65536 / FT_MAXT and leaves room for a co-resident kernel
#endif
template <bool VISCOUS, bool MERGED>
#ifdef FT_MAXNREG
__global__ void __maxnreg__(FT_MAXNREG) k_flowres
#else
__global__ void __launch_bounds__(FT_LB, FT_MINB) k_flowres
#endif
(Dims d, BlockDev b, FTile t, double rFil, int doDiss, int persistFw, int nw,
                                                        MffdEpi mf, const __grid_constant__ FTmaMaps maps, int zOff) {
    ADFB_PDL_SYNC();
    FSmem sm;
    sm.ring = ft_smem;
    sm.G = ft_smem + FT_NSLOT * FV_NUM * FT_S2;
    sm.EE = sm.G + FT_GP * FT_S0;
    sm.FX = sm.EE + FT_GP * FT_S0;
    unsigned long long* bars = reinterpret_cast<unsigned long long*>(sm.FX + (MERGED ? FT_NFLUX : FT_NFLUX_SPLIT) * FT_S0);   // 3 mbarriers
    const int tid = threadIdx.x;
    const FCtx x = ft_ctx(d, t, tid, blockIdx.x, blockIdx.y);
    const int ka = 2 + (blockIdx.z + zOff) * t.kChunk;   // zOff: the k chunks zOff .. of the slab pipeline; 0 otherwise
    const int kb = min(ka + t.kChunk - 1, d.kl);
    const int gi0 = blockIdx.x * (t.TX - 1), gj0 = blockIdx.y * (t.TY - 1);   // box index of the tile origin (i0-2, j0-2)
    const bool visc = VISCOUS && doDiss;
    int nUsed = 0;
#pragma unroll
    for (int v = 0; v < FV_NUM; v++) nUsed += ft_var_used(v, VISCOUS, doDiss) ? 1 : 0;
    const unsigned planeBytes = (unsigned)(nUsed * t.PX * t.PY * 8);

    if (t.useTma) {
        if (tid == 0) {
            for (int s = 0; s < FT_NSLOT; s++) ft_mbar_init(&bars[s], 1);
            asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
            asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
        }
        __syncthreads();
    }
    // asynchronous load of state plane kk into ring slot kk % FT_NSLOT
    auto load_plane = [&](int kk) {
        double* slot = sm.ring + (kk % FT_NSLOT) * (FV_NUM * FT_S2);
        if (t.useTma) {
            if (tid == 0) {
                unsigned long long* bar = &bars[kk % FT_NSLOT];
                ft_mbar_expect_tx(bar, planeBytes);
#pragma unroll
                for (int v = 0; v < FV_NUM; v++) {
                    if (!ft_var_used(v, VISCOUS, doDiss)) continue;
                    if (v == FV_AA) ft_tma_load_3d(slot + v * FT_S2, &maps.aa, gi0, gj0, kk, bar);
                    else if (v == FV_SS) ft_tma_load_3d(slot + v * FT_S2, &maps.ss, gi0, gj0, kk, bar);
                    else {
                        const int comp = v < 5 ? v : (v - 5 + nw);   // slab: w(0..nw-1), p, rlv, rev
                        ft_tma_load_3d(slot + v * FT_S2, &maps.slab, gi0, gj0, comp * d.NK + kk, bar);
                    }
                }
            }
        } else {
            const int np = t.PX * t.PY;
            for (int e = tid; e < np; e += t.nT) {
                const int py = e / t.PX, px = e - py * t.PX;
                const int gi = gi0 + px, gj = gj0 + py;
                const bool valid = gi <= d.ib && gj <= d.jb;
                const long long go = valid ? ((long long)gi + d.sJ * gj + d.sK * kk) : 0;
#pragma unroll
                for (int v = 0; v < FV_NUM; v++) {
                    if (!ft_var_used(v, VISCOUS, doDiss)) continue;
                    ft_cp_async8(slot + v * FT_S2 + e, ft_var_ptr(d, b, v) + go, valid);
                }
            }
            ft_cp_async_commit();
        }
    };
    auto wait_plane = [&](int kk) {
        if (t.useTma) ft_mbar_wait(&bars[kk % FT_NSLOT], (unsigned)(((kk - (ka - 1)) / FT_NSLOT) & 1));
        else ft_cp_async_wait_all();
    };

    load_plane(ka - 1);
    load_plane(ka);
    if (FT_NSLOT >= 3) load_plane(ka + 1);
    FRegs r;
    FStep st;
    ft_prologue_regs(c_prm, d, b, x, ka - 1, r, doDiss, VISCOUS);
    if ((FT_EARLY || (FT_AHEAD & (4 | 16))) && visc) ft_load_nodal(d, b, x, ka - 1, true, st.gn);
    wait_plane(ka - 1);
    wait_plane(ka);
    __syncthreads();

    for (int k = ka - 1; k <= kb; k++) {
        const double* A = sm.ring + (k % FT_NSLOT) * (FV_NUM * FT_S2);
        const double* B = sm.ring + ((k + 1) % FT_NSLOT) * (FV_NUM * FT_S2);
        const bool doIJ = k >= ka;
        if (FT_NSLOT == 2 && k > ka - 1) {   // two slots: plane k+1 was requested when plane k-1 retired, at the end of the previous step
            wait_plane(k + 1);
            __syncthreads();
        }
        ft_step_a<VISCOUS, MERGED>(d, b, t, x, k, kb, A, B, sm, r, st, doDiss, doIJ);
        __syncthreads();   // G / EE of this plane visible; the previous plane's flux exchange is over
        ft_step_b<VISCOUS, MERGED>(c_prm, d, b, t, x, k, kb, A, B, sm, r, st, rFil, doDiss, doIJ, 2);
        if (FT_NSLOT >= 3 && k + 2 <= kb + 1) wait_plane(k + 2);
        __syncthreads();   // fluxes visible; G / EE and the slot of plane k are free; (3 slots) plane k+2 has landed
        if (FT_NSLOT >= 3) { if (k + 3 <= kb + 1) load_plane(k + 3); }
        else if (k + 2 <= kb + 1) load_plane(k + 2);
        // bit 16: the nodal operands of the next plane are requested before the divergence of this one is formed
        if (!FT_EARLY && (FT_AHEAD & 16) && visc && k < kb) ft_load_nodal(d, b, x, k + 1, k + 1 < kb, st.gn);
        if (doIJ) ft_div<MERGED>(d, b, t, x, k, sm, r, st, rFil, persistFw, mf, c_prm.turbResScale);
#pragma unroll
        for (int l = 0; l < 10; l++) r.kprev[l] = st.kp[l];
    }
}

}  // namespace

// ---------------------------------------------------------------------------
// host: tensor maps + launch
typedef CUresult (*ft_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                 const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static ft_encode_fn ft_get_encoder() {
    static ft_encode_fn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
            fn = (ft_encode_fn)p;
        cudaGetLastError();
    }
    return fn;
}
// (NI, NJ, NK*ncomp) double tensor, box (PX, PY, 1); false when TMA cannot describe it (odd NI, no driver entry point)
static bool ft_make_map(CUtensorMap* m, const double* base, const Dims& d, int ncomp, const FTile& t) {
    ft_encode_fn enc = ft_get_encoder();
    if (!enc || (d.NI & 1) || (t.PX & 1) || t.PX > 256 || t.PY > 256) return false;   // 16-byte global strides and box rows
    const cuuint64_t dims[3] = {(cuuint64_t)d.NI, (cuuint64_t)d.NJ, (cuuint64_t)d.NK * ncomp};
    const cuuint64_t strides[2] = {(cuuint64_t)d.NI * 8, (cuuint64_t)d.NI * d.NJ * 8};
    const cuuint32_t box[3] = {(cuuint32_t)t.PX, (cuuint32_t)t.PY, 1};
    const cuuint32_t es[3] = {1, 1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT64, 3, (void*)base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int fused_mode() {   // ADFB_FUSED: 0 = off (k_nodal/k_faces/k_div), 1 = tile kernel with cp.async loads, 2 = with TMA (default)
    static int v = -1;
    if (v < 0) { const char* e = getenv("ADFB_FUSED"); v = e ? atoi(e) : 2; }
    return v;
}

// returns 0 on success, -1 when the tile kernel does not apply (caller uses the general kernels), > 0 on error
// kChunkForce > 0: that many planes per CTA instead of the wave-fitted chunk; zOff / zCount: only the k chunks zOff .. zOff+zCount-1
// (adfb_init raises the dynamic shared memory limit of every k_flowres instance to env.smemOptin)
static int launch_flowres_tile(const Dims& d, const BlockDev& b, const AdfbParams& prm, const LaunchEnv& env, int nw, double rFil, int doDiss,
                               bool merged, int persistFw, cudaStream_t stream, MffdEpi mf = MffdEpi{nullptr, 0}, int kChunkForce = 0,
                               int zOff = 0, int zCount = -1) {
    const bool viscous = prm.equations != ADFB_EULER;
    bool tma = fused_mode() >= 2 && !(d.NI & 1);
    FTile t = ftile_choose(d, tma, env.nSM);
    if (kChunkForce > 0) t.kChunk = kChunkForce;
    if (!merged) t.smemBytes += (size_t)(FT_NFLUX_SPLIT - FT_NFLUX) * FT_S0 * sizeof(double);   // central and dissipative fluxes exchanged apart
    if (!ftile_fits(t) || t.smemBytes > env.smemOptin) return -1;
    FTmaMaps maps;
    memset(&maps, 0, sizeof maps);
    if (tma) {
        // the state slab w(nw), p, rlv, rev is one allocation (adfb_block_create)
        tma = ft_make_map(&maps.slab, b.w, d, nw + 3, t) && ft_make_map(&maps.aa, b.aa, d, 1, t) && ft_make_map(&maps.ss, b.ss, d, 1, t);
        if (!tma) { t.useTma = 0; memset(&maps, 0, sizeof maps); }
    }
    const int nti = (d.nx + t.TX - 2) / (t.TX - 1), ntj = (d.ny + t.TY - 2) / (t.TY - 1), nkc = (d.nz + t.kChunk - 1) / t.kChunk;
    if (zCount < 0) zCount = nkc - zOff;
    if (zOff < 0 || zCount < 1 || zOff + zCount > nkc) return 1;
    dim3 grid(nti, ntj, zCount), block(t.nT);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = t.smemBytes; cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    cudaError_t e;
#define FT_LAUNCH(V, M) e = cudaLaunchKernelEx(&cfg, k_flowres<V, M>, d, b, t, rFil, doDiss, persistFw, nw, mf, maps, zOff)
    if (viscous) { if (merged) FT_LAUNCH(true, true); else FT_LAUNCH(true, false); }
    else { if (merged) FT_LAUNCH(false, true); else FT_LAUNCH(false, false); }
#undef FT_LAUNCH
    return e == cudaSuccess ? 0 : 1;
}
#endif  // __CUDACC__
