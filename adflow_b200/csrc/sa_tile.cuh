// sa_tile.cuh -- k-marching tile kernel for the SA row of the residual (sm_90a)
//
// k_sa forms dw(itu1) of the owned cells: saSource (blockette.F90:976-1168), saAdvection (:1392-1560), saViscous
// (:1170-1258) and the scaling (:623-627, :1872-1897), in the reference's order (source, advection k/j/i, diffusion k/j/i).
//
//   * a CTA owns a TX x TY tile of owned cell columns (thread (tx, ty) <-> column (i0+tx, j0+ty)) and marches a chunk of
//     k planes.  Per plane, shared memory holds u, v, w, nu = rlv/rho and vol of the tile with a one-cell halo, nt with a
//     two-cell halo (second-order advection), and si / sj of the tile's i / j faces.  Three plane buffers: planes k and
//     k+1 (the column's k+1 neighbour) are complete while plane k+2 arrives by cp.async, so the copies of a plane land
//     while the plane before it is formed instead of stalling every warp of the CTA at the barrier.  The column's own
//     operands (sk, d2Wall, volRef, iblank) are read one plane ahead into registers for the same reason.
//   * along k the column carries in registers what it needs of plane k-1 (u, v, w, nt, sk) and of k-2 (nt), and the
//     face quantities of the k face between k-1 and k, which the cell below formed as its upper face.
//   * every per-cell quotient (nu) is formed once, by the thread that copied the cell, once its copies have landed; ssum = s(c-sd) + s(c) is formed
//     from si / sj / sk with the same addition k_geom uses, so the row reads no ssum array.
//   * every expression keeps the operand order of the reference's loops, so the row is the one the per-cell form gave
//     (up to the FMA contractions the compiler picks).
//
// The per-thread phases are plain __host__ __device__ functions, so that tests/emul runs the identical code thread by
// thread on the CPU (tests/test_sa_emul.py) -- test infrastructure, never a product path.
#pragma once
#include "adfb_common.cuh"
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#if defined(__CUDACC__)
#define SHD __host__ __device__ __forceinline__
#else
#define SHD inline
#endif

// Shared-memory arrays are sized for the largest thread tile the chooser or a test uses: TX * TY <= SA_MAXT and the
// padded extents below (32 x 4 and 16 x 8 both fit).
#define SA_MAXT 128
#ifndef SA_MINB
#define SA_MINB 3        // resident CTAs per SM the register allocation is sized for (3 x 56 KB of shared memory fit an SM)
#endif
#define SA_NSLOT 3       // plane buffers: k, k+1 and the plane k+2 in flight while plane k is formed
#define SA_SF 204        // (TX+2) * (TY+2): u, v, w, nu (rlv until the plane is finished), vol, rho
#define SA_SN 288        // (TX+4) * (TY+4): nt
#define SA_SI 136        // (TX+1) * TY: si of the faces i0-1 .. i0+TX-1
#define SA_SJ 160        // TX * (TY+1): sj of the faces j0-1 .. j0+TY-1
#define SA_PLANE (6 * SA_SF + SA_SN + 3 * SA_SI + 3 * SA_SJ)   // doubles per plane buffer
#define SA_SMEM_BYTES ((size_t)SA_NSLOT * SA_PLANE * sizeof(double))
enum { SA_U = 0, SA_V, SA_W, SA_NU, SA_VOL, SA_RHO };

struct SaTile {
    int TX, TY;     // thread tile = owned cells per plane
    int nT;         // threads per CTA
    int kChunk;     // k planes per CTA
};

SHD bool sa_tile_fits(const SaTile& t) {
    return t.TX >= 1 && t.TY >= 1 && t.kChunk >= 1 && t.nT <= SA_MAXT && (t.TX + 2) * (t.TY + 2) <= SA_SF &&
           (t.TX + 4) * (t.TY + 4) <= SA_SN && (t.TX + 1) * t.TY <= SA_SI && t.TX * (t.TY + 1) <= SA_SJ;
}
static inline SaTile sa_tile_make(int TX, int TY, int kChunk) {
    SaTile t;
    t.TX = TX; t.TY = TY; t.kChunk = kChunk;
    t.nT = TX * TY;
    return t;
}
// Thread tile and k chunk for nPlanes owned planes of block d on nSM multiprocessors with ctasPerSM resident CTAs each:
// 32 x 4 or 16 x 8 (full 128-byte rows either way), whichever loads fewer halo cells over the block; then the longest
// k chunk that still fills every resident CTA slot once.  ADFB_SA_TILE=TX,TY,kChunk (tests) is taken instead when it fits
// the shared buffers, the chunk clamped to nPlanes; one that does not fit leaves the pick to the chooser.
static inline SaTile sa_tile_choose(const Dims& d, int nPlanes, int nSM, int ctasPerSM) {
    if (const char* e = getenv("ADFB_SA_TILE")) {
        int ox = 0, oy = 0, okc = 0;
        sscanf(e, "%d,%d,%d", &ox, &oy, &okc);
        if (ox >= 1 && oy >= 1 && ox <= SA_MAXT && oy <= SA_MAXT) {
            const SaTile o = sa_tile_make(ox, oy, okc < nPlanes ? okc : nPlanes);
            if (sa_tile_fits(o)) return o;
        }
    }
    const int shapes[2][2] = {{32, 4}, {16, 8}};
    long long best = -1;
    SaTile t = sa_tile_make(32, 4, 1);
    for (int s = 0; s < 2; s++) {
        const int TX = shapes[s][0], TY = shapes[s][1];
        const long long cost = (long long)((d.nx + TX - 1) / TX) * ((d.ny + TY - 1) / TY) * (TX + 2) * (TY + 2);
        if (best < 0 || cost < best) { best = cost; t = sa_tile_make(TX, TY, 1); }
    }
    const long long tiles = (long long)((d.nx + t.TX - 1) / t.TX) * ((d.ny + t.TY - 1) / t.TY);
    long long chunks = (long long)nSM * ctasPerSM / tiles;
    if (chunks < 1) chunks = 1;
    if (chunks > nPlanes) chunks = nPlanes;
    t.kChunk = (int)((nPlanes + chunks - 1) / chunks);
    if (t.kChunk < 1) t.kChunk = 1;
    return t;
}

// one plane buffer
struct SaPlane {
    double* f;    // [6][SA_SF]  u, v, w, nu, vol, rho at (a, b), a = -1 .. TX, b = -1 .. TY (cross only)
    double* nt;   // [SA_SN]     nt at a = -2 .. TX+1, b = -2 .. TY+1 (cross only; the outer ring with secondOrdTurb)
    double* si;   // [3][SA_SI]  si at a = -1 .. TX-1, b = 0 .. TY-1
    double* sj;   // [3][SA_SJ]  sj at a = 0 .. TX-1, b = -1 .. TY-1
};
SHD SaPlane sa_plane(double* base) {
    SaPlane p;
    p.f = base;
    p.nt = base + 6 * SA_SF;
    p.si = p.nt + SA_SN;
    p.sj = p.si + 3 * SA_SI;
    return p;
}
SHD int sa_fi(const SaTile& t, int a, int b) { return (a + 1) + (t.TX + 2) * (b + 1); }
SHD int sa_ni(const SaTile& t, int a, int b) { return (a + 2) + (t.TX + 4) * (b + 2); }
SHD int sa_ii(const SaTile& t, int a, int b) { return (a + 1) + (t.TX + 1) * b; }
SHD int sa_ji(const SaTile& t, int a, int b) { return a + t.TX * (b + 1); }

// One 8-byte copy global -> shared: asynchronous on the device (cp.async, completion per thread with sa_copy_wait), a plain
// store on the host.
SHD void sa_copy(double* dst, const double* src) {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
#else
    *dst = *src;
#endif
}
// Close the copies of one plane into a group; wait until at most `pending` of this thread's groups are still in flight.
SHD void sa_copy_commit() {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.commit_group;\n" ::: "memory");
#endif
}
template <int PENDING>
SHD void sa_copy_wait() {
#if defined(__CUDA_ARCH__)
    asm volatile("cp.async.wait_group %0;\n" ::"n"(PENDING) : "memory");
#endif
}

// The cells of plane buffer p that thread tid of nT loads: every nT-th cell of the (TX+4) x (TY+4) box around the tile with
// origin (i0, j0), cross only (no stencil reaches the corners); the outer ring holds nt only and only with secondOrdTurb.
// fn(c2d, a, b, ring1) gets the in-plane box offset of the cell and its tile coordinates.
template <typename Fn>
SHD void sa_plane_cells(const Dims& d, const SaTile& t, int tid, int i0, int j0, bool secondOrd, Fn&& fn) {
    const int PX = t.TX + 4, np = PX * (t.TY + 4);
    for (int e = tid; e < np; e += t.nT) {
        const int py = e / PX, px = e - py * PX;
        const int a = px - 2, bq = py - 2;
        const int gi = i0 + a, gj = j0 + bq;
        if (gi > d.ib || gj > d.jb) continue;   // past the box: only columns beyond il / jl would read it
        const bool inA = a >= 0 && a < t.TX, inB = bq >= 0 && bq < t.TY;
        if (!inA && !inB) continue;
        const bool ring1 = (inA && bq >= -1 && bq <= t.TY) || (inB && a >= -1 && a <= t.TX);
        if (!ring1 && !secondOrd) continue;
        fn(gi + (int)d.sJ * gj, a, bq, ring1);
    }
}

// Start the copies of plane kk into p (rlv goes to the nu slot; sa_finish_plane forms nu once the copies have landed).
SHD void sa_load_plane(const Dims& d, const BlockDev& b, const SaTile& t, int tid, int i0, int j0, int kk, bool secondOrd, const SaPlane& p) {
    const int N = (int)d.N, ck = (int)d.sK * kk;
    sa_plane_cells(d, t, tid, i0, j0, secondOrd, [&](int c2, int a, int bq, bool ring1) {
        const int c = c2 + ck;
        sa_copy(&p.nt[sa_ni(t, a, bq)], &b.w[5 * N + c]);
        if (!ring1) return;
        const int f = sa_fi(t, a, bq);
        sa_copy(&p.f[SA_U * SA_SF + f], &b.w[N + c]);
        sa_copy(&p.f[SA_V * SA_SF + f], &b.w[2 * N + c]);
        sa_copy(&p.f[SA_W * SA_SF + f], &b.w[3 * N + c]);
        sa_copy(&p.f[SA_NU * SA_SF + f], &b.rlv[c]);
        sa_copy(&p.f[SA_RHO * SA_SF + f], &b.w[c]);
        sa_copy(&p.f[SA_VOL * SA_SF + f], &b.vol[c]);
        if (bq >= 0 && bq < t.TY && a < t.TX) {
            const int q = sa_ii(t, a, bq);
#pragma unroll
            for (int m = 0; m < 3; m++) sa_copy(&p.si[m * SA_SI + q], &b.si[m * N + c]);
        }
        if (a >= 0 && a < t.TX && bq < t.TY) {
            const int q = sa_ji(t, a, bq);
#pragma unroll
            for (int m = 0; m < 3; m++) sa_copy(&p.sj[m * SA_SJ + q], &b.sj[m * N + c]);
        }
    });
}
// nu = rlv / rho of the cells this thread copied into p (its own copies have landed): once per cell and plane
SHD void sa_finish_plane(const Dims& d, const SaTile& t, int tid, int i0, int j0, bool secondOrd, const SaPlane& p) {
    sa_plane_cells(d, t, tid, i0, j0, secondOrd, [&](int, int a, int bq, bool ring1) {
        if (!ring1) return;
        const int f = sa_fi(t, a, bq);
        p.f[SA_NU * SA_SF + f] = p.f[SA_NU * SA_SF + f] / p.f[SA_RHO * SA_SF + f];
    });
}

// the quantities of one face that both of its cells use (saViscous): s * 2 / (vol_self + vol_other), the face averages
// of nt and nu.  Additions commute bit for bit, so the cell on the other side gets the same values.
struct SaFace { double x, y, z, nut, nu; };
SHD SaFace sa_face(double sx, double sy, double sz, double volSelf, double volOther, double ntSelf, double ntOther, double nuSelf,
                   double nuOther) {
    SaFace f;
    const double vf = 2.0 / (volSelf + volOther);
    f.x = sx * vf; f.y = sy * vf; f.z = sz * vf;
    f.nut = 0.5 * (ntOther + ntSelf);
    f.nu = 0.5 * (nuOther + nuSelf);
    return f;
}

// saAdvection, one direction (blockette.F90:1415-1560 for k; j, i analogous): nt at c-2sd .. c+2sd
SHD double sa_adv(bool secondOrd, double sx, double sy, double sz, double voli2, double ux, double uy, double uz, double ntm2, double ntm1,
                  double nt0, double ntp1, double ntp2) {
    const double xa = sx * voli2, ya = sy * voli2, za = sz * voli2;
    const double uu = xa * ux + ya * uy + za * uz;
    double dwtx;
    if (uu > 0.0) {
        if (secondOrd) {
            const double dwtm1 = ntm1 - ntm2;
            const double dwt = nt0 - ntm1;
            const double dwtp1 = ntp1 - nt0;
            dwtx = dwt;
            if (dwt * dwtp1 > 0.0) dwtx = dwtx + 0.5 * ((fabs(dwt) < fabs(dwtp1)) ? dwt : dwtp1);
            if (dwt * dwtm1 > 0.0) dwtx = dwtx - 0.5 * ((fabs(dwt) < fabs(dwtm1)) ? dwt : dwtm1);
        } else {
            dwtx = nt0 - ntm1;
        }
    } else {
        if (secondOrd) {
            const double dwtm1 = nt0 - ntm1;
            const double dwt = ntp1 - nt0;
            const double dwtp1 = ntp2 - ntp1;
            dwtx = dwt;
            if (dwt * dwtp1 > 0.0) dwtx = dwtx - 0.5 * ((fabs(dwt) < fabs(dwtp1)) ? dwt : dwtp1);
            if (dwt * dwtm1 > 0.0) dwtx = dwtx + 0.5 * ((fabs(dwt) < fabs(dwtm1)) ? dwt : dwtm1);
        } else {
            dwtx = ntp1 - nt0;
        }
    }
    return uu * dwtx;
}

// saViscous, one direction (blockette.F90:1197-1258 for k; j, i analogous): faces fm (c-sd side) and fp (c+sd side)
SHD double sa_visc(double cb2, double cb3Inv, const SaFace& fm, const SaFace& fp, double sx, double sy, double sz, double voli, double ntm,
                   double nt0, double ntp, double acc) {
    const double xa = 0.5 * sx * voli, ya = 0.5 * sy * voli, za = 0.5 * sz * voli;
    const double ttm = fm.x * xa + fm.y * ya + fm.z * za;
    const double ttp = fp.x * xa + fp.y * ya + fp.z * za;
    const double cnud = -cb2 * nt0 * cb3Inv;
    const double cam = ttm * cnud, cap = ttp * cnud;
    const double cdm = (fm.nu + (1.0 + cb2) * fm.nut) * ttm * cb3Inv;
    const double cdp = (fp.nu + (1.0 + cb2) * fp.nut) * ttp * cb3Inv;
    const double c1m = dmax_(cdm + cam, 0.0), c1p = dmax_(cdp + cap, 0.0);
    const double c10 = c1m + c1p;
    return acc + c1m * ntm - c10 * nt0 + c1p * ntp;
}

// saSource (blockette.F90:976-1168) from the velocity gradient sums gv[v][m] = sum over the six faces of +-q s_m
SHD double sa_source(const AdfbParams& P, double kar2Inv, const double (&gv)[3][3], double vol, double nt, double d2Wall, double nu) {
    const double fact = 0.25 / vol;
    const double sxx = 2.0 * fact * gv[0][0], syy = 2.0 * fact * gv[1][1], szz = 2.0 * fact * gv[2][2];
    const double sxy = fact * (gv[0][1] + gv[1][0]), sxz = fact * (gv[0][2] + gv[2][0]), syz = fact * (gv[1][2] + gv[2][1]);
    const double div2 = (2.0 * (1.0 / 3.0)) * ((sxx + syy + szz) * (sxx + syy + szz));
    const double strainMag2 = 2.0 * (sxy * sxy + sxz * sxz + syz * syz) + sxx * sxx + syy * syy + szz * szz;
    double sqrtProd;
    if (P.turbProd == ADFB_PROD_STRAIN) {
        sqrtProd = sqrt(dmax_(2.0 * strainMag2 - div2, 1.e-25));
    } else {
        const double vortx = 2.0 * fact * (gv[2][1] - gv[1][2]);
        const double vorty = 2.0 * fact * (gv[0][2] - gv[2][0]);
        const double vortz = 2.0 * fact * (gv[1][0] - gv[0][1]);
        sqrtProd = sqrt(vortx * vortx + vorty * vorty + vortz * vortz);
    }
    const double cv13 = P.rsaCv1 * P.rsaCv1 * P.rsaCv1;
    const double cw3 = P.rsaCw3;
    const double cw36 = (cw3 * cw3 * cw3) * (cw3 * cw3 * cw3);
    const double dist2Inv = 1.0 / (d2Wall * d2Wall);
    const double chi = nt / nu, chi2 = chi * chi, chi3 = chi * chi2;
    const double fv1 = chi3 / (chi3 + cv13);
    const double fv2 = 1.0 - chi / (1.0 + chi * fv1);
    double ft2 = 0.0;
    if (P.useft2SA) ft2 = P.rsaCt3 * exp(-P.rsaCt4 * chi2);
    double sst = sqrtProd + nt * fv2 * kar2Inv * dist2Inv;
    if (P.useRotationSA) sst = sst + P.rsaCrot * dmin_(0.0, sqrt(2.0 * strainMag2));
    sst = dmax_(sst, 1.e-10);
    double rr = nt * kar2Inv * dist2Inv / sst;
    rr = dmin_(rr, 10.0);
    const double rr2 = rr * rr, rr6 = rr2 * rr2 * rr2;
    const double gg = rr + P.rsaCw2 * (rr6 - rr);
    const double gg2 = gg * gg, gg6 = gg2 * gg2 * gg2;
    const double termFw = pow((1.0 + cw36) / (gg6 + cw36), 1.0 / 6.0);
    const double fwSa = gg * termFw;
    const double term1 = P.rsaCb1 * (1.0 - ft2) * sqrtProd * (P.approxSA ? 0.0 : 1.0);
    const double term2 = dist2Inv * (kar2Inv * P.rsaCb1 * ((1.0 - ft2) * fv2 + ft2) - P.rsaCw1 * fwSa);
    return (term1 + term2 * nt) * nt;
}

// what a column carries from one plane to the next
struct SaCarry {
    double u, v, w, nt;   // plane k-1
    double nt2;           // nt of plane k-2 (second-order advection)
    double sk[3];         // sk of plane k-1: the low k face of plane k
    SaFace fk;            // the k face between planes k-1 and k
};

// Thread context: the column (i, j) = (i0 + tx, j0 + ty); own = an owned column
struct SaCtx { int a, bq, i, j, c0; bool own; };
SHD SaCtx sa_ctx(const Dims& d, const SaTile& t, int tid, int i0, int j0) {
    SaCtx x;
    x.bq = tid / t.TX;
    x.a = tid - x.bq * t.TX;
    x.i = i0 + x.a; x.j = j0 + x.bq;
    x.own = x.i <= d.il && x.j <= d.jl;
    x.c0 = x.i + (int)d.sJ * x.j;
    return x;
}

// column prologue: the carried state for the first plane ka of the chunk, straight from global memory
SHD void sa_prologue(const Dims& d, const BlockDev& b, const SaCtx& x, int ka, bool secondOrd, SaCarry& cr) {
    if (!x.own) return;
    const int N = (int)d.N, sK = (int)d.sK;
    const int cm = x.c0 + sK * (ka - 1), c = cm + sK;
    cr.u = b.w[N + cm]; cr.v = b.w[2 * N + cm]; cr.w = b.w[3 * N + cm];
    cr.nt = b.w[5 * N + cm];
    cr.nt2 = secondOrd ? b.w[5 * N + cm - sK] : 0.0;
#pragma unroll
    for (int m = 0; m < 3; m++) cr.sk[m] = b.sk[m * N + cm];
    cr.fk = sa_face(cr.sk[0], cr.sk[1], cr.sk[2], b.vol[c], b.vol[cm], b.w[5 * N + c], cr.nt, b.rlv[c] / b.w[c], b.rlv[cm] / b.w[cm]);
}

// global-memory operands of the column's cell in plane k that are not in the plane buffers (read before the plane barrier)
struct SaOwn { double sk[3], ntp2, d2Wall, volRef; int iblank; };
SHD void sa_own_loads(const Dims& d, const BlockDev& b, const SaCtx& x, int k, bool secondOrd, SaOwn& o) {
    if (!x.own) return;
    const int N = (int)d.N, sK = (int)d.sK;
    const int c = x.c0 + sK * k;
#pragma unroll
    for (int m = 0; m < 3; m++) o.sk[m] = b.sk[m * N + c];
    o.ntp2 = secondOrd ? b.w[5 * N + c + 2 * sK] : 0.0;
    o.d2Wall = b.d2Wall[c];
    o.volRef = b.volRef[c];
    o.iblank = b.iblank[c];
}

// SA row of the column's cell in plane k: cur = plane k, nxt = plane k+1 (its centre only).  Returns dw(itu1) and
// advances the carry to plane k.
SHD double sa_cell(const AdfbParams& P, double cb3Inv, double kar2Inv, const SaTile& t, const SaCtx& x, const SaPlane& cur, const SaPlane& nxt,
                   const SaOwn& o, SaCarry& cr) {
    const bool so = P.secondOrdTurb != 0;
    const int a = x.a, bq = x.bq;
    const int f = sa_fi(t, a, bq), FJ = t.TX + 2;
    const int n = sa_ni(t, a, bq), NJ = t.TX + 4;
    const int qi = sa_ii(t, a, bq), qj = sa_ji(t, a, bq);
    const double* U = cur.f + SA_U * SA_SF;
    const double* V = cur.f + SA_V * SA_SF;
    const double* W = cur.f + SA_W * SA_SF;
    const double* NU = cur.f + SA_NU * SA_SF;
    const double* VOL = cur.f + SA_VOL * SA_SF;
    const double* NT = cur.nt;
    double r = 0.0;
    {   // saSource first, from the velocity gradient sums (only the carry and the column's own operands live across it)
        double gv[3][3];
#pragma unroll
        for (int v = 0; v < 3; v++) {
            const double* Q = cur.f + v * SA_SF;   // u, v, w
            const double qip = Q[f + 1], qim = Q[f - 1], qjp = Q[f + FJ], qjm = Q[f - FJ];
            const double qkp = nxt.f[v * SA_SF + f], qkm = v == 0 ? cr.u : v == 1 ? cr.v : cr.w;
#pragma unroll
            for (int m = 0; m < 3; m++)
                gv[v][m] = qip * cur.si[m * SA_SI + qi] - qim * cur.si[m * SA_SI + qi - 1] + qjp * cur.sj[m * SA_SJ + qj] -
                           qjm * cur.sj[m * SA_SJ + qj - t.TX] + qkp * o.sk[m] - qkm * cr.sk[m];
        }
        r = r + sa_source(P, kar2Inv, gv, VOL[f], NT[n], o.d2Wall, NU[f]);
    }
    const double vc = VOL[f], nu = NU[f], nt0 = NT[n];
    const double ux = U[f], uy = V[f], uz = W[f];
    // plane k+1 of the column
    const double ntP = nxt.nt[n], nuP = nxt.f[SA_NU * SA_SF + f], volP = nxt.f[SA_VOL * SA_SF + f];
    double siC[3], siM[3], sjC[3], sjM[3];
#pragma unroll
    for (int m = 0; m < 3; m++) {
        siC[m] = cur.si[m * SA_SI + qi]; siM[m] = cur.si[m * SA_SI + qi - 1];
        sjC[m] = cur.sj[m * SA_SJ + qj]; sjM[m] = cur.sj[m * SA_SJ + qj - t.TX];
    }
    const double rblank = dmax_((double)o.iblank, 0.0);
    // ssum = s(c-sd) + s(c), as k_geom forms it
    double ssK[3], ssJ[3], ssI[3];
#pragma unroll
    for (int m = 0; m < 3; m++) { ssI[m] = siM[m] + siC[m]; ssJ[m] = sjM[m] + sjC[m]; ssK[m] = cr.sk[m] + o.sk[m]; }
    const double voli2 = 0.5 / vc;
    r = r - sa_adv(so, ssK[0], ssK[1], ssK[2], voli2, ux, uy, uz, cr.nt2, cr.nt, nt0, ntP, o.ntp2);
    r = r - sa_adv(so, ssJ[0], ssJ[1], ssJ[2], voli2, ux, uy, uz, so ? NT[n - 2 * NJ] : 0.0, NT[n - NJ], nt0, NT[n + NJ], so ? NT[n + 2 * NJ] : 0.0);
    r = r - sa_adv(so, ssI[0], ssI[1], ssI[2], voli2, ux, uy, uz, so ? NT[n - 2] : 0.0, NT[n - 1], nt0, NT[n + 1], so ? NT[n + 2] : 0.0);

    const double cb2 = P.rsaCb2;
    const double voli = 1.0 / vc;
    // k: the low face came up from the cell below; the high face goes up to the cell above
    const SaFace kHi = sa_face(o.sk[0], o.sk[1], o.sk[2], vc, volP, nt0, ntP, nu, nuP);
    r = sa_visc(cb2, cb3Inv, cr.fk, kHi, ssK[0], ssK[1], ssK[2], voli, cr.nt, nt0, ntP, r);
    {
        const SaFace lo = sa_face(sjM[0], sjM[1], sjM[2], vc, VOL[f - FJ], nt0, NT[n - NJ], nu, NU[f - FJ]);
        const SaFace hi = sa_face(sjC[0], sjC[1], sjC[2], vc, VOL[f + FJ], nt0, NT[n + NJ], nu, NU[f + FJ]);
        r = sa_visc(cb2, cb3Inv, lo, hi, ssJ[0], ssJ[1], ssJ[2], voli, NT[n - NJ], nt0, NT[n + NJ], r);
    }
    {
        const SaFace lo = sa_face(siM[0], siM[1], siM[2], vc, VOL[f - 1], nt0, NT[n - 1], nu, NU[f - 1]);
        const SaFace hi = sa_face(siC[0], siC[1], siC[2], vc, VOL[f + 1], nt0, NT[n + 1], nu, NU[f + 1]);
        r = sa_visc(cb2, cb3Inv, lo, hi, ssI[0], ssI[1], ssI[2], voli, NT[n - 1], nt0, NT[n + 1], r);
    }
    // advance the carry to plane k
    cr.u = ux; cr.v = uy; cr.w = uz;
    cr.nt2 = cr.nt; cr.nt = nt0;
#pragma unroll
    for (int m = 0; m < 3; m++) cr.sk[m] = o.sk[m];
    cr.fk = kHi;
    return -o.volRef * r * rblank;
}

// ===========================================================================
// device side
#if defined(__CUDACC__)
namespace {

// k_sa: SA row of the owned cells i 2..il, j 2..jl, k 2+kOff .. min(kl, kTop) (kOff / kTop: the slab pipeline's planes;
// 0 / INT_MAX: all of them).  Grid: (i tiles, j tiles, k chunks of the plane range).
__global__ void __launch_bounds__(SA_MAXT, SA_MINB) k_sa(Dims d, BlockDev b, SaTile t, MffdEpi mf, int kOff, int kTop) {
    extern __shared__ __align__(16) double sa_smem[];   // SA_NSLOT plane buffers
    const int tid = threadIdx.x;
    const int i0 = 2 + blockIdx.x * t.TX, j0 = 2 + blockIdx.y * t.TY;
    const int ka = 2 + kOff + blockIdx.z * t.kChunk;
    const int kb = min(ka + t.kChunk - 1, min(d.kl, kTop));
    const bool so = c_prm.secondOrdTurb != 0;
    const double cb3Inv = c_fheat[3] /* 1 / rsaCb3 */, kar2Inv = c_fheat[4] /* 1 / rsaK**2 */;
    const SaCtx x = sa_ctx(d, t, tid, i0, j0);
    auto slot = [&](int k) { return sa_plane(sa_smem + ((k - ka) % SA_NSLOT) * SA_PLANE); };
    // planes ka and ka+1 in flight; the column's carried state and its own operands of plane ka meanwhile
    sa_load_plane(d, b, t, tid, i0, j0, ka, so, slot(ka));
    sa_copy_commit();
    sa_load_plane(d, b, t, tid, i0, j0, ka + 1, so, slot(ka + 1));
    sa_copy_commit();
    SaCarry cr;
    sa_prologue(d, b, x, ka, so, cr);
    SaOwn oNext;
    sa_own_loads(d, b, x, ka, so, oNext);
    sa_copy_wait<1>();
    sa_finish_plane(d, t, tid, i0, j0, so, slot(ka));
    for (int k = ka; k <= kb; k++) {
        // plane k+2 into the buffer plane k-1 left (the last one a column needs is kb+1); it lands while plane k is formed
        if (k + 2 <= kb + 1) sa_load_plane(d, b, t, tid, i0, j0, k + 2, so, slot(k + 2));
        sa_copy_commit();
        const SaOwn o = oNext;
        if (k < kb) sa_own_loads(d, b, x, k + 1, so, oNext);
        sa_copy_wait<1>();   // this thread's copies of plane k+1 have landed
        sa_finish_plane(d, t, tid, i0, j0, so, slot(k + 1));
        __syncthreads();     // planes k and k+1 are complete in shared memory
        if (x.own) {
            const double dwv = sa_cell(c_prm, cb3Inv, kar2Inv, t, x, slot(k), slot(k + 1), o, cr);
            const int c = x.c0 + (int)d.sK * k;
            b.dw[5 * d.N + c] = dwv;
            if (mf.rec) mffd_epilogue(mf, d, x.i, x.j, k, 5, dwv, o.volRef, c_prm.turbResScale);
        }
        __syncthreads();     // plane k's buffer is free for plane k+3
    }
}

}  // namespace

// The SA row of planes 2+kOff .. min(kl, kTop): tile and k chunk from the block and the device (sa_tile_choose).
static int launch_sa(const Dims& d, const BlockDev& b, const LaunchEnv& env, MffdEpi mf, int kOff, int kTop, cudaStream_t stream) {
    const int nPlanes = (kTop < d.kl ? kTop : d.kl) - (2 + kOff) + 1;
    if (nPlanes <= 0) return 0;
    const SaTile t = sa_tile_choose(d, nPlanes, env.nSM > 0 ? env.nSM : 1, env.saCtasPerSM > 0 ? env.saCtasPerSM : 1);
    const dim3 g((d.nx + t.TX - 1) / t.TX, (d.ny + t.TY - 1) / t.TY, (nPlanes + t.kChunk - 1) / t.kChunk);
    return (int)launch_kernel(K_SA, false, g, t.nT, SA_SMEM_BYTES, stream, k_sa, d, b, t, mf, kOff, kTop);
}
#endif
