// smoother_kernels.cuh -- boundary-condition, Runge-Kutta and residual-averaging kernels
//
//   k_bc_level  : applyAllTurbBCThisBlock (src/turbulence/turbBCRoutines.F90:49-236) and applyAllBC_block
//                 (src/solver/BCRoutines.F90:57-222) for the BC classes symmetry, polar symmetry, adiabatic /
//                 isothermal NS wall, far field, sub- / supersonic in- and outflow, extrapolation and Euler wall.
//                 launch_bc_levels issues the reference's ordered (subface, phase) items as levels of mutually
//                 independent items, one launch per level, so the edge / corner halos keep the reference's order.
//   k_rk_scale / k_rk_update : executeRkStage (src/solver/smoothers.F90:90-382)
//   k_resavg_rfl / k_resavg_eps / k_resavg_sweep / k_resavg_lines : residualAveraging (src/solver/residuals.F90:1785-2080)
//   k_wall_forces : wallIntegrationFace, forces and moments (src/solver/surfaceIntegrations.F90:406-881)
#pragma once
#include "adfb_common.cuh"
#include <math.h>

struct FaceDev {
    long long off[4];  // plane 0 (2nd halo) .. 3 (2nd interior), setBCPointers utils.F90:881
    long long sa, sb;  // in-plane strides
    int icBeg, icEnd, jcBeg, jcEnd;
    int bcType;
    const double *norm, *rface, *uSlip, *TNSWall;
    const double *ps, *rho, *velx, *vely, *velz, *ptInlet, *ttInlet, *htInlet, *fxd, *fyd, *fzd, *turbInlet;
    int inletTreatment;
    long long xoff;   // node plane of the boundary face (polar symmetry reads the mesh)
    int bLo, bHi;     // clip of the second in-plane index (the slab pipeline applies the i / j faces plane range by plane range)
};

static FaceDev make_face(const Dims& d, const AdfbSubface& sf) {
    FaceDev f;
    switch (sf.faceId) {
        case ADFB_IMIN: f.off[0] = 0; f.off[1] = 1; f.off[2] = 2; f.off[3] = 3; f.sa = d.sJ; f.sb = d.sK; break;
        case ADFB_IMAX: f.off[0] = d.ib; f.off[1] = d.ie; f.off[2] = d.il; f.off[3] = d.nx; f.sa = d.sJ; f.sb = d.sK; break;
        case ADFB_JMIN: f.off[0] = 0; f.off[1] = d.sJ; f.off[2] = 2 * d.sJ; f.off[3] = 3 * d.sJ; f.sa = 1; f.sb = d.sK; break;
        case ADFB_JMAX: f.off[0] = d.jb * d.sJ; f.off[1] = d.je * d.sJ; f.off[2] = d.jl * d.sJ; f.off[3] = d.ny * d.sJ; f.sa = 1; f.sb = d.sK; break;
        case ADFB_KMIN: f.off[0] = 0; f.off[1] = d.sK; f.off[2] = 2 * d.sK; f.off[3] = 3 * d.sK; f.sa = 1; f.sb = d.sJ; break;
        default: f.off[0] = d.kb * d.sK; f.off[1] = d.ke * d.sK; f.off[2] = d.kl * d.sK; f.off[3] = d.nz * d.sK; f.sa = 1; f.sb = d.sJ; break;
    }
    f.icBeg = sf.icBeg; f.icEnd = sf.icEnd; f.jcBeg = sf.jcBeg; f.jcEnd = sf.jcEnd;
    f.bLo = -(1 << 30); f.bHi = 1 << 30;
    f.bcType = sf.bcType;
    f.norm = sf.norm; f.rface = sf.rface; f.uSlip = sf.uSlip; f.TNSWall = sf.TNSWall;
    f.ps = sf.ps; f.rho = sf.rho; f.velx = sf.velx; f.vely = sf.vely; f.velz = sf.velz;
    f.ptInlet = sf.ptInlet; f.ttInlet = sf.ttInlet; f.htInlet = sf.htInlet;
    f.fxd = sf.flowXdirInlet; f.fyd = sf.flowYdirInlet; f.fzd = sf.flowZdirInlet; f.turbInlet = sf.turbInlet;
    f.inletTreatment = sf.subsonicInletTreatment;
    f.xoff = (sf.faceId == ADFB_IMIN || sf.faceId == ADFB_JMIN || sf.faceId == ADFB_KMIN) ? f.off[1] : f.off[2];
    return f;
}

namespace {

__device__ __forceinline__ void bc_etot(const BlockDev& b, long long N, long long c) {
    const double ovgm1 = 1.0 / (c_prm.gammaInf - 1.0);
    const double r = b.w[c], u = b.w[N + c], v = b.w[2 * N + c], w = b.w[3 * N + c];
    b.w[4 * N + c] = ovgm1 * b.p[c] + 0.5 * r * (u * u + v * v + w * w);
}
// extrapolate2ndHalo, src/solver/BCRoutines.F90:1870-1918
__device__ __forceinline__ void bc_extrap2(const BlockDev& b, long long N, long long c0, long long c1, long long c2) {
    double r0 = 2.0 * b.w[c1] - b.w[c2];
    r0 = dmax_(0.5 * b.w[c1], r0);
    b.w[c0] = r0;
    b.w[N + c0] = 2.0 * b.w[N + c1] - b.w[N + c2];
    b.w[2 * N + c0] = 2.0 * b.w[2 * N + c1] - b.w[2 * N + c2];
    b.w[3 * N + c0] = 2.0 * b.w[3 * N + c1] - b.w[3 * N + c2];
    b.p[c0] = dmax_(0.5 * b.p[c1], 2.0 * b.p[c1] - b.p[c2]);
    if (c_prm.equations != ADFB_EULER) b.rlv[c0] = b.rlv[c1];
    if (c_prm.equations == ADFB_RANS) b.rev[c0] = b.rev[c1];
    bc_etot(b, N, c0);
}

__device__ __forceinline__ void bc_turb_cell(const Dims& d, const BlockDev& b, const FaceDev& f, int ia, int jb, int secondHalo) {
    const long long N = d.N;
    const long long q = ia * f.sa + jb * f.sb;
    const long long c0 = f.off[0] + q, c1 = f.off[1] + q, c2 = f.off[2] + q;
    const long long na = f.icEnd - f.icBeg + 1, nb = f.jcEnd - f.jcBeg + 1;
    const long long o = (ia - f.icBeg) + na * (jb - f.jcBeg);
    double bmt = 0.0, bvt = 0.0;
    const bool wall = f.bcType == ADFB_BC_NSWALL_ADIABATIC || f.bcType == ADFB_BC_NSWALL_ISOTHERMAL;
    if (wall) bmt = 1.0;
    else if (f.bcType == ADFB_BC_FARFIELD) {
        const double dot = f.norm[o] * c_prm.wInf[1] + f.norm[o + na * nb] * c_prm.wInf[2] + f.norm[o + 2 * na * nb] * c_prm.wInf[3] -
                           (f.rface ? f.rface[o] : 0.0);
        if (dot > 0.0) bmt = -1.0; else bvt = c_prm.wInf[5];
    } else if (f.bcType == ADFB_BC_SUBSONIC_INFLOW || f.bcType == ADFB_BC_SUPERSONIC_INFLOW) {
        bvt = 2.0 * (f.turbInlet ? f.turbInlet[o] : 0.0);   // bcTurbInflow, turbBCRoutines.F90:460-515
        bmt = 1.0;
    } else bmt = -1.0;  // symm, Euler wall, extrapolation, outflow: zero gradient
    double* nt = b.w + 5 * N;
    double v1 = bvt;
    v1 = v1 - bmt * nt[c2];
    nt[c1] = v1;
    const double r1 = wall ? -b.rev[c2] : b.rev[c2];
    b.rev[c1] = r1;
    if (secondHalo) { nt[c0] = v1; b.rev[c0] = r1; }
}

// phase: 1 = symmetry first halo, 2 = symmetry second halo, 0 = everything else.
// Register form: the interior states are read once, the halo states are built in registers (total energy and the
// second-halo extrapolation included) and stored once -- the reference's routines re-read what they just wrote
// (computeEtot, extrapolate2ndHalo: BCRoutines.F90:1870-1918), which on the device is a chain of dependent global
// round trips per subface; the arithmetic and its order are unchanged.
struct BcCellState { double r, u, v, w, e, p, rlv, rev; };
__device__ __forceinline__ void bc_flow_cell(const Dims& d, const BlockDev& b, const FaceDev& f, int ia, int jb, int secondHalo, int phase) {
    const long long N = d.N;
    const long long q = ia * f.sa + jb * f.sb;
    const long long c0 = f.off[0] + q, c1 = f.off[1] + q, c2 = f.off[2] + q, c3 = f.off[3] + q;
    const long long na = f.icEnd - f.icBeg + 1, nb = f.jcEnd - f.jcBeg + 1;
    const long long o = (ia - f.icBeg) + na * (jb - f.jcBeg);
    const double n1 = f.norm ? f.norm[o] : 0.0, n2 = f.norm ? f.norm[o + na * nb] : 0.0, n3 = f.norm ? f.norm[o + 2 * na * nb] : 0.0;
    const double rface = f.rface ? f.rface[o] : 0.0;
    const bool viscous = c_prm.equations != ADFB_EULER, eddy = c_prm.equations == ADFB_RANS;
    const double gam = c_prm.gammaInf;
    double* w = b.w;
    auto load = [&](long long c) {
        BcCellState s;
        s.r = w[c]; s.u = w[N + c]; s.v = w[2 * N + c]; s.w = w[3 * N + c]; s.e = w[4 * N + c]; s.p = b.p[c];
        s.rlv = viscous ? b.rlv[c] : 0.0;
        s.rev = eddy ? b.rev[c] : 0.0;
        return s;
    };
    auto store = [&](long long c, const BcCellState& s) {
        w[c] = s.r; w[N + c] = s.u; w[2 * N + c] = s.v; w[3 * N + c] = s.w; w[4 * N + c] = s.e; b.p[c] = s.p;
        if (viscous) b.rlv[c] = s.rlv;
        if (eddy) b.rev[c] = s.rev;
    };
    auto etot = [&](BcCellState& s) {   // computeEtot (cpConstant)
        const double ovgm1 = 1.0 / (c_prm.gammaInf - 1.0);
        s.e = ovgm1 * s.p + 0.5 * s.r * (s.u * s.u + s.v * s.v + s.w * s.w);
    };
    if (f.bcType == ADFB_BC_SYMM || f.bcType == ADFB_BC_SYMMPOLAR) {
        // bcSymm1stHalo / bcSymm2ndHalo, BCRoutines.F90:223-340; bcSymmPolar1stHalo / 2ndHalo, :332-486
        const BcCellState si = load(phase == 1 ? c2 : c3);
        BcCellState sh = si;
        if (f.bcType == ADFB_BC_SYMM) {
            const double vn = 2.0 * (si.u * n1 + si.v * n2 + si.w * n3);
            sh.u = si.u - vn * n1; sh.v = si.v - vn * n2; sh.w = si.w - vn * n3;
        } else {
            const long long nA = f.xoff + q, nB = f.xoff + (ia - 1) * f.sa + (jb - 1) * f.sb;
            double nnx = b.x[nA] - b.x[nB], nny = b.x[N + nA] - b.x[N + nB], nnz = b.x[2 * N + nA] - b.x[2 * N + nB];
            double tmp = 1.0 / sqrt(nnx * nnx + nny * nny + nnz * nnz);
            nnx = nnx * tmp; nny = nny * tmp; nnz = nnz * tmp;
            tmp = 2.0 * (si.u * nnx + si.v * nny + si.w * nnz);
            sh.u = tmp * nnx - si.u; sh.v = tmp * nny - si.v; sh.w = tmp * nnz - si.w;
        }
        store(phase == 1 ? c1 : c0, sh);
        return;
    }
    const BcCellState s2 = load(c2);
    BcCellState s1 = s2;   // rlv1 = rlv2, rev1 = rev2 unless changed below
    switch (f.bcType) {
        case ADFB_BC_NSWALL_ADIABATIC: {  // bcNSWallAdiabatic, BCRoutines.F90:489-578
            double us1 = 0.0, us2 = 0.0, us3 = 0.0;
            if (f.uSlip) { us1 = f.uSlip[o]; us2 = f.uSlip[o + na * nb]; us3 = f.uSlip[o + 2 * na * nb]; }
            s1.u = -s2.u + 2.0 * us1; s1.v = -s2.v + 2.0 * us2; s1.w = -s2.w + 2.0 * us3;
            s1.rev = -s2.rev;
            if (c_prm.wallBCConstantPressure || b.coarse) {   // BCRoutines.F90:550,642: coarse levels use constant pressure
                s1.p = s2.p;
            } else {
                double p1 = 2.0 * s2.p - b.p[c3];
                if (p1 <= 0.0) p1 = s2.p;
                s1.p = p1;
            }
            break;
        }
        case ADFB_BC_NSWALL_ISOTHERMAL: {  // bcNSWallIsoThermal, BCRoutines.F90:579-691
            double us1 = 0.0, us2 = 0.0, us3 = 0.0;
            if (f.uSlip) { us1 = f.uSlip[o]; us2 = f.uSlip[o + na * nb]; us3 = f.uSlip[o + 2 * na * nb]; }
            const double tw = f.TNSWall[o];
            const double t2 = s2.p / (c_prm.RGas * s2.r);
            double t1 = 2.0 * tw - t2;
            t1 = dmax_(0.5 * tw, t1);
            t1 = dmin_(2.0 * tw, t1);
            double p1;
            if (c_prm.wallBCConstantPressure || b.coarse) {
                p1 = s2.p;
            } else {
                p1 = 2.0 * s2.p - b.p[c3];
                if (p1 <= 0.0) p1 = s2.p;
            }
            s1.p = p1;
            s1.r = p1 / (c_prm.RGas * t1);
            s1.u = -s2.u + 2.0 * us1; s1.v = -s2.v + 2.0 * us2; s1.w = -s2.w + 2.0 * us3;
            s1.rev = -s2.rev;
            break;
        }
        case ADFB_BC_EXTRAP:
        case ADFB_BC_SUPERSONIC_OUTFLOW: {  // bcExtrap, BCRoutines.F90:1479-1570
            double fw2 = 2.0, fw3 = -1.0;   // extrap: linear; supersonic outflow: outflowTreatment
            if (f.bcType == ADFB_BC_SUPERSONIC_OUTFLOW && !c_prm.outflowLinearExtrapol) { fw2 = 1.0; fw3 = 0.0; }
            const double r3 = w[c3], u3 = w[N + c3], v3 = w[2 * N + c3], w3 = w[3 * N + c3], p3 = b.p[c3];
            double r1 = fw2 * s2.r + fw3 * r3;
            r1 = dmax_(0.5 * s2.r, r1);
            s1.r = r1;
            s1.u = fw2 * s2.u + fw3 * u3;
            s1.v = fw2 * s2.v + fw3 * v3;
            s1.w = fw2 * s2.w + fw3 * w3;
            double p1 = fw2 * s2.p + fw3 * p3;
            p1 = dmax_(0.5 * s2.p, p1);
            s1.p = p1;
            break;
        }
        case ADFB_BC_SUBSONIC_OUTFLOW: {  // bcSubsonicOutflow, BCRoutines.F90:693-802
            const double pExit = f.ps[o];
            const double ovg = 1.0 / gam, ovgm1 = 1.0 / (gam - 1.0);
            const double pInt = s2.p;
            const double r = 1.0 / s2.r;
            const double a2 = gam * pInt * r;
            double a = sqrt(a2);
            const double ue = s2.u, ve = s2.v, we = s2.w;
            const double qne = ue * n1 + ve * n2 + we * n3;
            const double ss = pInt * pow(r, gam);
            const double ac = qne + 2.0 * a * ovgm1;
            const double r1 = pow(pExit / ss, ovg);
            s1.r = r1;
            s1.p = pExit;
            a = sqrt(gam * pExit / r1);
            const double qnh = ac - 2.0 * a * ovgm1;
            s1.u = ue + (qnh - qne) * n1;
            s1.v = ve + (qnh - qne) * n2;
            s1.w = we + (qnh - qne) * n3;
            break;
        }
        case ADFB_BC_SUBSONIC_INFLOW: {  // bcSubsonicInflow, BCRoutines.F90:804-1061 (cpConstant)
            const double gm1 = gam - 1.0, ovgm1 = 1.0 / gm1;
            const double r = 1.0 / s2.r;
            double a2 = gam * s2.p * r;
            double beta = s2.u * n1 + s2.v * n2 + s2.w * n3 + 2.0 * ovgm1 * sqrt(a2);
            if (f.inletTreatment == 1) {   // totalConditions
                const double govgm1 = gam / (gam - 1.0);
                const double ptot = f.ptInlet[o], ttot = f.ttInlet[o], htot = f.htInlet[o];
                const double ssx = f.fxd[o], ssy = f.fyd[o], ssz = f.fzd[o];
                double scaleFact = 1.0;
                if (c_prm.hScalingInlet) scaleFact = sqrt(htot / (r * (s2.e + s2.p)));
                beta = beta * scaleFact;
                double q2 = s2.u * s2.u + s2.v * s2.v + s2.w * s2.w;
                const double a2tot = gm1 * (htot - r * (s2.e + s2.p) + 0.5 * q2) + a2;
                const double alpha = n1 * ssx + n2 * ssy + n3 * ssz;
                const double aa2 = 0.5 * gm1 * alpha * alpha + 1.0;
                const double bb = -gm1 * alpha * beta;
                const double cc = 0.5 * gm1 * beta * beta - 2.0 * ovgm1 * a2tot;
                double dd = bb * bb - 4.0 * aa2 * cc;
                dd = sqrt(dmax_(0.0, dd));
                double qq = (-bb + dd) / (2.0 * aa2);
                qq = dmax_(0.0, qq);
                q2 = qq * qq;
                a2 = a2tot - 0.5 * gm1 * q2;
                double m2 = q2 / a2;
                m2 = dmin_(1.0, m2);
                q2 = m2 * a2;
                qq = sqrt(q2);
                a2 = a2tot - 0.5 * gm1 * q2;
                s1.u = qq * ssx; s1.v = qq * ssy; s1.w = qq * ssz;
                const double ts = a2 / (gam * c_prm.RGas);
                const double ratio = pow(ts / ttot, govgm1);
                s1.p = ptot * ratio;
                s1.r = (ptot * ratio) / (c_prm.RGas * ts);
            } else {                        // massFlow
                const double rho = f.rho[o], velx = f.velx[o], vely = f.vely[o], velz = f.velz[o];
                a2 = 0.5 * gm1 * (beta - velx * n1 - vely * n2 - velz * n3);
                a2 = dmax_(0.0, a2);
                a2 = a2 * a2;
                s1.p = rho * a2 / gam;
                s1.r = rho; s1.u = velx; s1.v = vely; s1.w = velz;
            }
            break;
        }
        case ADFB_BC_SUPERSONIC_INFLOW: {  // bcSupersonicInflow, BCRoutines.F90:1411-1477
            s1.r = f.rho[o]; s1.u = f.velx[o]; s1.v = f.vely[o]; s1.w = f.velz[o];
            s1.p = f.ps[o];
            etot(s1);
            store(c1, s1);
            if (secondHalo) store(c0, s1);   // same prescribed state, rlv/rev of the first halo, same total energy
            return;
        }
        case ADFB_BC_FARFIELD: {  // bcFarfield, BCRoutines.F90:1282-1396
            const double gm1 = gam - 1.0, ovgm1 = 1.0 / gm1;
            const double r0 = 1.0 / c_prm.wInf[0], u0 = c_prm.wInf[1], v0 = c_prm.wInf[2], w0 = c_prm.wInf[3];
            const double c0s = c_fheat[6];   // sqrt(gam * pInfCorr * r0)           } evaluated once per parameter set on the
            const double s0 = c_fheat[5];    // pow(wInf[0], gam) / pInfCorr        } device (k_param_consts): same bits
            const double qn0 = u0 * n1 + v0 * n2 + w0 * n3;
            const double vn0 = qn0 - rface;
            const double rho2 = s2.r;
            const double re = 1.0 / rho2, ue = s2.u, ve = s2.v, we = s2.w;
            const double qne = ue * n1 + ve * n2 + we * n3;
            const double p2 = s2.p;
            const double ce = sqrt(gam * p2 * re);
            double ac1, ac2;
            if (vn0 > -c0s) ac1 = qne + 2.0 * ovgm1 * ce; else ac1 = qn0 + 2.0 * ovgm1 * c0s;
            if (vn0 > c0s) ac2 = qne - 2.0 * ovgm1 * ce; else ac2 = qn0 - 2.0 * ovgm1 * c0s;
            const double qnf = 0.5 * (ac1 + ac2);
            const double cf = 0.25 * (ac1 - ac2) * gm1;
            double uf, vf, wf, sfv;
            if (vn0 > 0.0) {
                uf = ue + (qnf - qne) * n1; vf = ve + (qnf - qne) * n2; wf = we + (qnf - qne) * n3;
                sfv = pow(rho2, gam) / p2;
            } else {
                uf = u0 + (qnf - qn0) * n1; vf = v0 + (qnf - qn0) * n2; wf = w0 + (qnf - qn0) * n3;
                sfv = s0;
            }
            const double cc = cf * cf / gam;
            const double r1 = pow(sfv * cc, ovgm1);
            s1.r = r1; s1.u = uf; s1.v = vf; s1.w = wf;
            s1.p = r1 * cc;
            break;
        }
        case ADFB_BC_EULERWALL: {  // bcEulerWall, BCRoutines.F90:1063-1280 (constant / linear pressure)
            const double grad = (c_prm.reserved || b.coarse) ? 0.0 : b.p[c3] - s2.p;   // BCRoutines.F90:1100
            s1.p = dmax_(s2.p - grad, 0.0);
            const double vn = 2.0 * (rface - s2.u * n1 - s2.v * n2 - s2.w * n3);
            s1.u = s2.u + vn * n1; s1.v = s2.v + vn * n2; s1.w = s2.w + vn * n3;
            break;
        }
        default: return;
    }
    etot(s1);
    store(c1, s1);
    if (secondHalo) {   // extrapolate2ndHalo, BCRoutines.F90:1870-1918
        BcCellState s0;
        s0.r = dmax_(0.5 * s1.r, 2.0 * s1.r - s2.r);
        s0.u = 2.0 * s1.u - s2.u;
        s0.v = 2.0 * s1.v - s2.v;
        s0.w = 2.0 * s1.w - s2.w;
        s0.p = dmax_(0.5 * s1.p, 2.0 * s1.p - s2.p);
        s0.rlv = s1.rlv; s0.rev = s1.rev;
        etot(s0);
        store(c0, s0);
    }
}

// up to ADFB_BC_MAXSUB subfaces of a block, passed by value to one launch of the SA wall terms (k_sa_bmt); blocks with more
// subfaces take one launch per ADFB_BC_MAXSUB of them
#define ADFB_BC_MAXSUB 12
struct BcList {
    int n;
    int la[ADFB_BC_MAXSUB], lb[ADFB_BC_MAXSUB];   // owned upper index of the two in-plane directions (il/jl/kl)
    FaceDev f[ADFB_BC_MAXSUB];
};

// One LEVEL of the ordered BC sweep.  Two items of the reference's ordered list (subface, kind) can only influence each other
// when they touch common cells: subfaces on faces of different index directions (they share the edge / corner halos of
// the block), or the same cells of one face (turbulence BC and flow BC of one subface both write the eddy-viscosity halo).
// Subfaces on opposite faces, disjoint subfaces of one face and the two symmetry phases of one subface read and write
// disjoint cells.  Items are given the level 1 + max(level of the earlier items they conflict with); the items of one level
// run in one launch (blockIdx.z = item), the levels in the reference's order -- every conflicting pair keeps its order,
// so the halos are the reference's bit for bit, in about half as many launches as one per item.
#define ADFB_BC_LEVEL_MAX 8
struct BcLevel {   // passed by value: the face descriptors sit in the constant bank, no dependent global load before the state loads
    int n;
    int kind[ADFB_BC_LEVEL_MAX];
    FaceDev f[ADFB_BC_LEVEL_MAX];
};
__global__ void __launch_bounds__(128) k_bc_level(Dims d, BlockDev b, const __grid_constant__ BcLevel lv, int secondHalo) {
    ADFB_PDL_SYNC();
    const FaceDev& f = lv.f[blockIdx.z];
    const int kind = lv.kind[blockIdx.z];
    const int ia = blockIdx.x * blockDim.x + threadIdx.x + f.icBeg;
    const int jb = blockIdx.y * blockDim.y + threadIdx.y + f.jcBeg;
    if (ia > f.icEnd || jb > f.jcEnd || jb < f.bLo || jb > f.bHi) return;
    if (kind == 3) bc_turb_cell(d, b, f, ia, jb, secondHalo);
    else bc_flow_cell(d, b, f, ia, jb, secondHalo, kind);
}

// ---------------------------------------------------------------------------
// executeRkStage part 1: dw *= cfl*etaRK(stage)*dtl, smoothers.F90:196-218
__global__ void __launch_bounds__(256) k_rk_scale(Dims d, BlockDev b, double tmp) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const long long c = ADFB_IDX(i, j, k), N = d.N;
    const double dt = tmp * b.dtl[c];
#pragma unroll
    for (int l = 0; l < 5; l++) b.dw[l * N + c] = b.dw[l * N + c] * dt;
}

// executeRkStage part 2 (smoothers.F90:298-354): conservative update -> primitive,
// clips, then computeEtotBlock + computeLamViscosity + computeEddyViscosity fused.
// scaleDt != 0 folds part 1 in (used when no residual averaging runs in between).
// fromCurrent != 0: the DADI update, which starts from the current w, p instead of wn, pn (smoothers.F90:614-640)
__global__ void __launch_bounds__(256) k_rk_update(Dims d, BlockDev b, int scaleDt, double tmp, int nw, int fromCurrent) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const long long c = ADFB_IDX(i, j, k), N = d.N;
    double dw[5];
#pragma unroll
    for (int l = 0; l < 5; l++) dw[l] = b.dw[l * N + c];
    if (scaleDt) {
        const double dt = tmp * b.dtl[c];
#pragma unroll
        for (int l = 0; l < 5; l++) { dw[l] = dw[l] * dt; b.dw[l * N + c] = dw[l]; }
    }
    const double gm1 = c_prm.gammaInf - 1.0;
    const double rho = b.w[c], u = b.w[N + c], v = b.w[2 * N + c], w = b.w[3 * N + c], e = b.w[4 * N + c];
    double ovr = 1.0 / rho;
    const double v2 = u * u + v * v + w * w;
    const double dp = (ovr * b.p[c] + 0.0 - gm1 * (ovr * e - v2)) * dw[0] + gm1 * (dw[4] - u * dw[1] - v * dw[2] - w * dw[3]);
    const double rn = fromCurrent ? rho : b.wn[c];
    double rnew = rn - dw[0];
    rnew = dmax_(rnew, 1.e-4 * c_prm.rhoInf);
    const double ru = rn * (fromCurrent ? u : b.wn[N + c]) - dw[1];
    const double rv = rn * (fromCurrent ? v : b.wn[2 * N + c]) - dw[2];
    const double rw = rn * (fromCurrent ? w : b.wn[3 * N + c]) - dw[3];
    ovr = 1.0 / rnew;
    const double un = ovr * ru, vn = ovr * rv, wn_ = ovr * rw;
    double pnew = (fromCurrent ? b.p[c] : b.pn[c]) - dp;
    pnew = dmax_(pnew, 1.e-4 * c_prm.pInfCorr);
    b.w[c] = rnew; b.w[N + c] = un; b.w[2 * N + c] = vn; b.w[3 * N + c] = wn_;
    b.p[c] = pnew;
    b.w[4 * N + c] = (1.0 / gm1) * pnew + 0.5 * rnew * (un * un + vn * vn + wn_ * wn_);
    if (c_prm.equations == ADFB_EULER) return;
    const double T = pnew / (c_prm.RGas * rnew);
    const double rlv = c_prm.muSuth * ((c_prm.TSuth + c_prm.SSuth) / (T + c_prm.SSuth)) * pow(T / c_prm.TSuth, 1.5);
    b.rlv[c] = rlv;
    if (c_prm.equations != ADFB_RANS || nw < 6) return;
    const double rnuSA = b.w[5 * N + c] * rnew;
    const double chi = rnuSA / rlv;
    const double chi3 = chi * chi * chi;
    const double cv13 = c_prm.rsaCv1 * c_prm.rsaCv1 * c_prm.rsaCv1;
    b.rev[c] = chi3 / (chi3 + cv13) * rnuSA;
}

// ---------------------------------------------------------------------------
// residualAveraging, one direction (residuals.F90:1850-1927 i, :1929-1993 j, :1995-2078 k).
// One thread per grid line; n owned cells along the line (stride sd); the two other
// owned index ranges are spanned by the grid (q1 fastest).  epz/d/t live in scratch
// slots 0..2 of the block (same box indexing).
__device__ __forceinline__ double ra_rfl(const BlockDev& b, const Dims& d, long long c, double plim) {
    const double* p = b.p;
    const double p0 = p[c];
    const double dpi = fabs(p[c + 1] - 2.0 * p0 + p[c - 1]) / (p[c + 1] + 2.0 * p0 + p[c - 1] + plim);
    const double dpj = fabs(p[c + d.sJ] - 2.0 * p0 + p[c - d.sJ]) / (p[c + d.sJ] + 2.0 * p0 + p[c - d.sJ] + plim);
    const double dpk = fabs(p[c + d.sK] - 2.0 * p0 + p[c - d.sK]) / (p[c + d.sK] + 2.0 * p0 + p[c - d.sK] + plim);
    return 1.0 / (1.0 + 2.0 * (dpi + dpj + dpk));
}
// residualAveraging (residuals.F90:1785-2080), split so that only the recurrences are serial.
// Workspace b.flux: slot 0 rfl (pressure switch), 1..3 epz of the i, j, k direction (both one pass per
// call, one thread per cell), 4..8 the forward-swept residuals, 9..13 d(i) per variable.
__global__ void __launch_bounds__(256) k_resavg_rfl(Dims d, BlockDev b) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const long long c = ADFB_IDX(i, j, k);
    b.flux[c] = ra_rfl(b, d, c, 0.001 * c_prm.pInfCorr);
}
// epz(i) = 1/4 smoop max(r^2 - 1, 0) max(iblank, 0), r = rfl0 (rfl(i) + rfl(i+1)), for i < l; epz(l) = 0
__global__ void __launch_bounds__(256) k_resavg_eps(Dims d, BlockDev b, double rfl0) {
    ADFB_PDL_SYNC();
    const int i = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int j = blockIdx.y * blockDim.y + threadIdx.y + 2;
    const int k = blockIdx.z * blockDim.z + threadIdx.z + 2;
    if (i > d.il || j > d.jl || k > d.kl) return;
    const long long c = ADFB_IDX(i, j, k), N = d.N;
    const double* rfl = b.flux;
    const double smoop = c_prm.smoop, r0 = rfl[c], rblank = dmax_((double)b.iblank[c], 0.0);
    double e = 0.0, r;
    if (i < d.il) { r = rfl0 * (r0 + rfl[c + 1]); e = 0.25 * smoop * dmax_(r * r - 1.0, 0.0) * rblank; }
    b.flux[N + c] = e;
    e = 0.0;
    if (j < d.jl) { r = rfl0 * (r0 + rfl[c + d.sJ]); e = 0.25 * smoop * dmax_(r * r - 1.0, 0.0) * rblank; }
    b.flux[2 * N + c] = e;
    e = 0.0;
    if (k < d.kl) { r = rfl0 * (r0 + rfl[c + d.sK]); e = 0.25 * smoop * dmax_(r * r - 1.0, 0.0) * rblank; }
    b.flux[3 * N + c] = e;
}
// one thread per line and variable m = blockIdx.z: t(i) = 1/(1 + epz(i) + epz(i-1) - epz(i-1) d(i-1)),
// d(i) = t(i) epz(i), forward sweep dw(i) = t(i) (dw(i) + epz(i-1) dw(i-1)), back substitution
__global__ void __launch_bounds__(64) k_resavg_sweep(Dims d, BlockDev b, int dir, long long sd, int n, long long s1, int n1,
                                                     long long s2, int n2) {
    ADFB_PDL_SYNC();
    const int q1 = blockIdx.x * blockDim.x + threadIdx.x + 2;
    const int q2 = blockIdx.y * blockDim.y + threadIdx.y + 2;
    if (q1 > n1 + 1 || q2 > n2 + 1) return;
    const long long N = d.N;
    const long long base = q1 * s1 + q2 * s2;
    const int m = blockIdx.z;
    const double* __restrict__ epzA = b.flux + (1 + dir) * N;
    double* __restrict__ fo = b.flux + (4 + m) * N;
    double* __restrict__ dA = b.flux + (9 + m) * N;
    double* __restrict__ dw = b.dw + m * N;
    const int l = n + 1;
    double dwm = 0.0, epzm = 0.0, dm = 0.0;  // epz(1) = d(1) = 0
    constexpr int CH = 8;  // chunked walk: loads of a chunk first, then the serial chain
    for (int i0 = 2; i0 <= l; i0 += CH) {
        double eq[CH], wq[CH];
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int i = i0 + u;
            if (i <= l) { const long long c = base + i * sd; eq[u] = epzA[c]; wq[u] = dw[c]; }
        }
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int i = i0 + u;
            if (i <= l) {
                const long long c = base + i * sd;
                const double epz = eq[u];
                const double t = 1.0 / (1.0 + epz + epzm - epzm * dm);
                const double dd = t * epz;
                const double v = t * (wq[u] + epzm * dwm);
                fo[c] = v; dA[c] = dd;
                dwm = v; epzm = epz; dm = dd;
            }
        }
    }
    dw[base + l * sd] = dwm;
    for (int i0 = n; i0 >= 2; i0 -= CH) {
        double fq[CH], dq[CH];
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int i = i0 - u;
            if (i >= 2) { const long long c = base + i * sd; fq[u] = fo[c]; dq[u] = dA[c]; }
        }
#pragma unroll
        for (int u = 0; u < CH; u++) {
            const int i = i0 - u;
            if (i >= 2) {
                const double v = fq[u] + dq[u] * dwm;
                dw[base + i * sd] = v;
                dwm = v;
            }
        }
    }
}

// residualAveraging along one direction with the whole solve in shared memory: a CTA takes LPC grid lines and the 5
// variables (LPC x 5 threads).
//   A  all threads copy the lines' epz and dw into shared memory, consecutive threads along the direction that is
//      contiguous in HBM (the line itself for i lines, the line index for j / k lines): every global access coalesced
//   B  one thread per line factorises: t(i) = 1 / (1 + epz(i) + epz(i-1) - epz(i-1) d(i-1)), d(i) = t(i) epz(i) -- once
//      per line instead of once per (line, variable), the only chain with a division
//   C  one thread per (line, variable): forward sweep v(i) = t(i) (dw(i) + epz(i-1) v(i-1)) and back substitution
//      v(i) += d(i) v(i+1), in place in shared memory (two-FMA chains)
//   D  coalesced copy back to dw
// HBM traffic 88 B per cell and direction (epz + dw in, dw out) instead of 192 B with the forward-swept values in
// global memory, and the serial walks never wait for HBM.  Same operations on the same operands as k_resavg_sweep.
#define ADFB_RA_THREADS 768   // copy phases: enough loads in flight to fill the SM's share of HBM bandwidth
static const size_t kResavgSmemMax = 220 * 1024;   // dynamic shared memory a CTA may take
// lines are numbered id = (q1 - 2) + n1 (q2 - 2); a CTA takes LPC consecutive ids (LPC is sized on the host so that the
// grid is one wave of the SMs), LP = padded pitch of the shared arrays (odd: conflict free along and across the lines)
__global__ void __launch_bounds__(ADFB_RA_THREADS) k_resavg_lines(Dims d, BlockDev b, int dir, long long sd, int n, long long s1, int n1,
                                                                  long long s2, int n2, int LPC, int LP) {
    ADFB_PDL_SYNC();
    extern __shared__ double ra_sm[];
    double* T = ra_sm;                          // [n][LP]
    double* D = T + (size_t)n * LP;
    double* E = D + (size_t)n * LP;
    double* F = E + (size_t)n * LP;             // [5][n][LP]
    long long* lineBase = reinterpret_cast<long long*>(F + (size_t)5 * n * LP);   // [LPC] box offset of cell 0 of the line minus 2 sd
    const int tid = threadIdx.x, nT = blockDim.x;
    const int lane = tid % LPC, m = tid / LPC;   // solve phases: the first LPC * 5 threads
    const int id0 = blockIdx.x * LPC;
    const int nLines = min(LPC, n1 * n2 - id0);
    if (tid < nLines) {
        const int id = id0 + tid;
        lineBase[tid] = (long long)(id % n1 + 2) * s1 + (long long)(id / n1 + 2) * s2 + 2 * sd;
    }
    __syncthreads();
    const long long N = d.N;
    const double* __restrict__ epzA = b.flux + (1 + dir) * N;
    const bool alongLine = sd == 1;   // i lines: the cells of a line are contiguous
    // ---- A: load
    const int total = n * nLines;
    for (int e = tid; e < total; e += nT) {
        const int i = alongLine ? e % n : e / nLines, ln = alongLine ? e / n : e % nLines;
        const long long c = lineBase[ln] + i * sd;
        E[i * LP + ln] = epzA[c];
#pragma unroll
        for (int v = 0; v < 5; v++) F[((size_t)v * n + i) * LP + ln] = b.dw[v * N + c];
    }
    __syncthreads();
    // ---- B: factorisation, one thread per line
    if (m == 0 && lane < nLines) {
        double epzm = 0.0, dm = 0.0;   // epz(1) = d(1) = 0
#pragma unroll 8
        for (int i = 0; i < n; i++) {
            const double epz = E[i * LP + lane];
            const double t = 1.0 / (1.0 + epz + epzm - epzm * dm);
            const double dd = t * epz;
            T[i * LP + lane] = t; D[i * LP + lane] = dd;
            epzm = epz; dm = dd;
        }
    }
    __syncthreads();
    // ---- C: forward sweep and back substitution of one (line, variable)
    if (m < 5 && lane < nLines) {
        double* f = F + (size_t)m * n * LP + lane;
        double dwm = 0.0, epzm = 0.0;
#pragma unroll 8
        for (int i = 0; i < n; i++) {
            const double v = T[i * LP + lane] * (f[i * LP] + epzm * dwm);
            f[i * LP] = v;
            dwm = v; epzm = E[i * LP + lane];
        }
#pragma unroll 8
        for (int i = n - 2; i >= 0; i--) {
            const double v = f[i * LP] + D[i * LP + lane] * dwm;
            f[i * LP] = v;
            dwm = v;
        }
    }
    __syncthreads();
    // ---- D: store
    for (int e = tid; e < total; e += nT) {
        const int i = alongLine ? e % n : e / nLines, ln = alongLine ? e / n : e % nLines;
        const long long c = lineBase[ln] + i * sd;
#pragma unroll
        for (int v = 0; v < 5; v++) b.dw[v * N + c] = F[((size_t)v * n + i) * LP + ln];
    }
}

// lines per CTA of the shared-memory line kernels: one wave of one CTA per SM if the lines fit, else the largest count
// that fits (nArr arrays of n x LP doubles + the line table)
static int lines_per_cta(long long nLinesTotal, int n, int nArr, int maxLpc, size_t lim, int nSM, int* LPout, size_t* bytesOut) {
    auto bytes = [&](int lpc) { const int LP = lpc | 1; return (size_t)nArr * n * LP * sizeof(double) + (size_t)lpc * sizeof(long long); };
    int lpc = (int)((nLinesTotal + nSM - 1) / nSM);
    if (lpc < 4) lpc = (int)(nLinesTotal < 4 ? nLinesTotal : 4);
    if (lpc > maxLpc) lpc = maxLpc;
    while (lpc > 1 && bytes(lpc) > lim) lpc--;
    if (bytes(lpc) > lim) return 0;
    *LPout = lpc | 1;
    *bytesOut = bytes(lpc);
    return lpc;
}

// wallIntegrationFace, force and moment part (src/solver/surfaceIntegrations.F90:406-881): one CTA per wall
// subface; every thread sums its face cells in index order, then a fixed-order tree reduction, so the result
// is run-to-run reproducible.  acc = Fp(3), Fv(3), Mp(3), Mv(3).  sib: the subface's surface iblank (BCData%iblank,
// extents icBeg:icEnd x jcBeg:jcEnd), NULL == 1.
__global__ void __launch_bounds__(256) k_wall_forces(Dims d, BlockDev b, FaceDev f, const int32_t* sib, int dir, int isMin, int la, int lb,
                                                     int viscWall, double r0, double r1, double r2, double pRef, double* acc) {
    ADFB_PDL_SYNC();
    __shared__ double sh[12][256];
    const long long N = d.N;
    const double fact = isMin ? -1.0 : 1.0;
    const double* s = dir == 0 ? b.si : (dir == 1 ? b.sj : b.sk);
    const int a0 = f.icBeg < 2 ? 2 : f.icBeg, a1 = f.icEnd > la ? la : f.icEnd;
    const int b0 = f.jcBeg < 2 ? 2 : f.jcBeg, b1 = f.jcEnd > lb ? lb : f.jcEnd;
    const int na = a1 - a0 + 1, nb = b1 - b0 + 1;
    const int nfa = f.icEnd - f.icBeg + 1;
    const long long pstride = dir == 0 ? d.NJ : d.NI;
    const double* tau = b.wallTau + ((long long)(dir * 2 + (isMin ? 0 : 1)) * 9) * b.wallP;
    double v[12];
#pragma unroll
    for (int q = 0; q < 12; q++) v[q] = 0.0;
    for (int idx = threadIdx.x; idx < na * nb; idx += blockDim.x) {
        const int ia = a0 + idx % na, jb = b0 + idx / na;
        const long long q = ia * f.sa + jb * f.sb;
        const long long c1 = f.off[1] + q, c2 = f.off[2] + q;
        const long long cf = isMin ? c1 : c2;
        const double blk = sib ? dmax_((double)sib[(ia - f.icBeg) + nfa * (jb - f.jcBeg)], 0.0) : 1.0;
        double xc[3];
#pragma unroll
        for (int m = 0; m < 3; m++) {
            const double* xm = b.x + m * N;
            xc[m] = 0.25 * (xm[cf - f.sa - f.sb] + xm[cf - f.sb] + xm[cf - f.sa] + xm[cf]);
        }
        const double rx = xc[0] - r0, ry = xc[1] - r1, rz = xc[2] - r2;
        const double s1 = s[cf], s2 = s[N + cf], s3 = s[2 * N + cf];
        const double pm1 = fact * (0.5 * (b.p[c2] + b.p[c1]) - c_prm.pInf) * pRef;
        double fx = pm1 * s1, fy = pm1 * s2, fz = pm1 * s3;
        v[0] += fx * blk; v[1] += fy * blk; v[2] += fz * blk;
        v[6] += (ry * fz - rz * fy) * blk; v[7] += (rz * fx - rx * fz) * blk; v[8] += (rx * fy - ry * fx) * blk;
        if (viscWall) {
            const long long pi = ia + pstride * jb;
            const double txx = tau[pi], tyy = tau[b.wallP + pi], tzz = tau[2 * b.wallP + pi], txy = tau[3 * b.wallP + pi],
                         txz = tau[4 * b.wallP + pi], tyz = tau[5 * b.wallP + pi];
            fx = -fact * (txx * s1 + txy * s2 + txz * s3) * pRef;
            fy = -fact * (txy * s1 + tyy * s2 + tyz * s3) * pRef;
            fz = -fact * (txz * s1 + tyz * s2 + tzz * s3) * pRef;
            v[3] += fx * blk; v[4] += fy * blk; v[5] += fz * blk;
            v[9] += (ry * fz - rz * fy) * blk; v[10] += (rz * fx - rx * fz) * blk; v[11] += (rx * fy - ry * fx) * blk;
        }
    }
#pragma unroll
    for (int q = 0; q < 12; q++) sh[q][threadIdx.x] = v[q];
    __syncthreads();
    for (int w = blockDim.x / 2; w > 0; w >>= 1) {
        if ((int)threadIdx.x < w) {
#pragma unroll
            for (int q = 0; q < 12; q++) sh[q][threadIdx.x] += sh[q][threadIdx.x + w];
        }
        __syncthreads();
    }
    if (threadIdx.x < 12) acc[threadIdx.x] += sh[threadIdx.x][0];
}

}  // namespace

// the reference's ordered list of (subface, kind) items of one BC sweep (applyAllTurbBCThisBlock, then applyAllBC_block in its
// BC-class order: BCRoutines.F90:81-216); kind 3 = turbulence BC, 1 / 2 = symmetry first / second halo, 0 = the other classes
static std::vector<std::pair<int, int>> bc_ordered_items(const std::vector<AdfbSubface>& subs, int secondHalo, int withTurb, int withFlow) {
    std::vector<std::pair<int, int>> it;
    const int n = (int)subs.size();
    if (withTurb) for (int q = 0; q < n; q++) it.emplace_back(q, 3);
    if (withFlow) {
        for (int q = 0; q < n; q++) if (subs[q].bcType == ADFB_BC_SYMM) it.emplace_back(q, 1);
        if (secondHalo) for (int q = 0; q < n; q++) if (subs[q].bcType == ADFB_BC_SYMM) it.emplace_back(q, 2);
        for (int q = 0; q < n; q++) if (subs[q].bcType == ADFB_BC_SYMMPOLAR) it.emplace_back(q, 1);
        if (secondHalo) for (int q = 0; q < n; q++) if (subs[q].bcType == ADFB_BC_SYMMPOLAR) it.emplace_back(q, 2);
        const int order[8][2] = {{ADFB_BC_NSWALL_ADIABATIC, -1}, {ADFB_BC_NSWALL_ISOTHERMAL, -1}, {ADFB_BC_FARFIELD, -1},
                                 {ADFB_BC_SUBSONIC_OUTFLOW, -1}, {ADFB_BC_SUBSONIC_INFLOW, -1}, {ADFB_BC_EXTRAP, ADFB_BC_SUPERSONIC_OUTFLOW},
                                 {ADFB_BC_EULERWALL, -1}, {ADFB_BC_SUPERSONIC_INFLOW, -1}};
        for (int gq = 0; gq < 8; gq++)
            for (int q = 0; q < n; q++)
                if (subs[q].bcType == order[gq][0] || subs[q].bcType == order[gq][1]) it.emplace_back(q, 0);
    }
    return it;
}
// can two items of the ordered list touch common cells?
static bool bc_items_conflict(const std::vector<AdfbSubface>& subs, std::pair<int, int> a, std::pair<int, int> c) {
    const AdfbSubface& A = subs[a.first];
    const AdfbSubface& C = subs[c.first];
    if ((A.faceId - 1) / 2 != (C.faceId - 1) / 2) return true;    // faces of different directions share edge / corner halos
    if (A.faceId != C.faceId) return false;                       // opposite faces
    if (a.first == c.first) {                                     // one subface: the symmetry phases are disjoint, the rest is not
        const bool symPhases = (a.second == 1 && c.second == 2) || (a.second == 2 && c.second == 1);
        return !symPhases;
    }
    const bool apart = A.icEnd < C.icBeg || C.icEnd < A.icBeg || A.jcEnd < C.jcBeg || C.jcEnd < A.jcBeg;
    return !apart;                                                // subfaces of one face: disjoint unless their ranges overlap
}
// The ordered BC sweep as levels of mutually independent items (k_bc_level).  bLo / bHi clip the k index of the i- and j-face
// subfaces, kFaces selects the k-face subfaces (1 = kMin, 2 = kMax): the slab pipeline of adfb_form_function applies the
// sweep plane range by plane range -- an i/j-face cell touches its own k plane only, a k-face cell the planes 0..3 or
// kl-1..kb, so every conflicting pair of items still meets inside one slab, in the reference's order.
static int launch_bc_levels(const Dims& d, const BlockDev& b, const std::vector<AdfbSubface>& subs, int secondHalo, int withTurb, int withFlow,
                            cudaStream_t s, int bLo = -(1 << 30), int bHi = 1 << 30, int kFaces = 3) {
    const std::vector<std::pair<int, int>> items = bc_ordered_items(subs, secondHalo, withTurb, withFlow);
    if (items.empty()) return (int)cudaGetLastError();   // still reports a pending launch error
    std::vector<int> level(items.size(), 1);
    int nLevels = 1;
    for (size_t q = 0; q < items.size(); q++) {
        for (size_t r = 0; r < q; r++)
            if (level[r] >= level[q] && bc_items_conflict(subs, items[r], items[q])) level[q] = level[r] + 1;
        if (level[q] > nLevels) nLevels = level[q];
    }
    for (int l = 1; l <= nLevels; l++) {
        BcLevel lv;
        lv.n = 0;
        int ma = 1, mb = 1;
        auto flush = [&]() {
            if (!lv.n) return;
            launch_kernel(K_BC, true, dim3((ma + 31) / 32, (mb + 3) / 4, (unsigned)lv.n), dim3(32, 4), 0, s, k_bc_level, d, b, lv, secondHalo);
            lv.n = 0; ma = 1; mb = 1;
        };
        for (size_t q = 0; q < items.size(); q++) {
            if (level[q] != l) continue;
            const AdfbSubface& sf = subs[items[q].first];
            const bool kFace = sf.faceId == ADFB_KMIN || sf.faceId == ADFB_KMAX;
            if (kFace && !(kFaces & (sf.faceId == ADFB_KMIN ? 1 : 2))) continue;
            FaceDev f = make_face(d, sf);
            if (!kFace) {
                f.bLo = bLo; f.bHi = bHi;
                if (sf.jcEnd < bLo || sf.jcBeg > bHi) continue;   // nothing of this subface in the plane range
            }
            lv.f[lv.n] = f; lv.kind[lv.n] = items[q].second; lv.n++;
            ma = std::max(ma, sf.icEnd - sf.icBeg + 1);
            mb = std::max(mb, sf.jcEnd - sf.jcBeg + 1);
            if (lv.n == ADFB_BC_LEVEL_MAX) flush();   // more independent items than one launch carries: any order
        }
        flush();
    }
    return (int)cudaGetLastError();
}
// the subfaces subs[q0], subs[q0 + 1], ... of a block, at most ADFB_BC_MAXSUB of them
static BcList make_bc_list(const Dims& d, const std::vector<AdfbSubface>& subs, size_t q0) {
    BcList L;
    memset(&L, 0, sizeof(BcList));
    L.n = (int)std::min(subs.size() - q0, (size_t)ADFB_BC_MAXSUB);
    for (int q = 0; q < L.n; q++) {
        L.f[q] = make_face(d, subs[q0 + q]);
        const int face = subs[q0 + q].faceId;
        L.la[q] = (face == ADFB_IMIN || face == ADFB_IMAX) ? d.jl : d.il;
        L.lb[q] = (face == ADFB_KMIN || face == ADFB_KMAX) ? d.jl : d.kl;
    }
    return L;
}

static int launch_residual_averaging(const Dims& d, const BlockDev& b, const AdfbParams& prm, const LaunchEnv& env, cudaStream_t s) {
    const double rfl0 = 0.5 * prm.cfl / prm.cflLimit;
    {
        dim3 tb(32, 4, 2);
        dim3 g((d.nx + 31) / 32, (d.ny + 3) / 4, (d.nz + 1) / 2);
        launch_kernel(K_RK, true, g, tb, 0, s, k_resavg_rfl, d, b);
        launch_kernel(K_RK, true, g, tb, 0, s, k_resavg_eps, d, b, rfl0);
    }
    dim3 tb(32, 2);
    auto run = [&](int dir, long long sd, int n, long long s1, int n1, long long s2, int n2) {
        if (n <= 1) return;
        int LP = 0; size_t smem = 0;
        const int lpc = lines_per_cta((long long)n1 * n2, n, 8, ADFB_RA_THREADS / 5, kResavgSmemMax, env.nSM, &LP, &smem);
        if (lpc)
            launch_kernel(K_RK, true, (unsigned)(((long long)n1 * n2 + lpc - 1) / lpc), ADFB_RA_THREADS, smem, s, k_resavg_lines, d, b, dir, sd, n,
                          s1, n1, s2, n2, lpc, LP);
        else   // not even one line fits into shared memory (n >= 3520 cells)
            launch_kernel(K_RK, true, dim3((n1 + 31) / 32, (n2 + 1) / 2, 5), tb, 0, s, k_resavg_sweep, d, b, dir, sd, n, s1, n1, s2, n2);
    };
    run(0, 1, d.nx, d.sJ, d.ny, d.sK, d.nz);
    run(1, d.sJ, d.ny, 1, d.nx, d.sK, d.nz);
    run(2, d.sK, d.nz, 1, d.nx, d.sJ, d.ny);
    return (int)cudaGetLastError();
}

static int launch_rk_update(const Dims& d, const BlockDev& b, const AdfbParams& prm, const LaunchEnv& env, int rkStage, cudaStream_t s,
                            int nwOverride = 0) {
    const double tmp = prm.cfl * prm.etaRK[rkStage - 1];
    const bool smooth = prm.resAveraging == 1 || (prm.resAveraging == 2 && (rkStage % 2) == 1);
    dim3 tb(32, 4, 2);
    dim3 g((d.nx + 31) / 32, (d.ny + 3) / 4, (d.nz + 1) / 2);
    const int nw = nwOverride ? nwOverride : (prm.equations == ADFB_RANS ? 6 : 5);   // 5: eddy viscosity frozen (coarse levels)
    if (smooth) {
        launch_kernel(K_RK, true, g, tb, 0, s, k_rk_scale, d, b, tmp);
        if (launch_residual_averaging(d, b, prm, env, s)) return 1;
        launch_kernel(K_RK, true, g, tb, 0, s, k_rk_update, d, b, 0, tmp, nw, 0);
    } else {
        launch_kernel(K_RK, true, g, tb, 0, s, k_rk_update, d, b, 1, tmp, nw, 0);
    }
    return (int)cudaGetLastError();
}

// state update of executeDADIStep (smoothers.F90:595-650) after computedwDADI
static int launch_dadi_update(const Dims& d, const BlockDev& b, const AdfbParams& prm, const LaunchEnv& env, cudaStream_t s, int nwOverride = 0) {
    if (prm.resAveraging == 1)  // rkStage == 0 in the DADI smoother: `alternate` never smooths (smoothers.F90:461-469)
        if (launch_residual_averaging(d, b, prm, env, s)) return 1;
    dim3 tb(32, 4, 2);
    dim3 g((d.nx + 31) / 32, (d.ny + 3) / 4, (d.nz + 1) / 2);
    launch_kernel(K_RK, true, g, tb, 0, s, k_rk_update, d, b, 0, 0.0, nwOverride ? nwOverride : (prm.equations == ADFB_RANS ? 6 : 5), 1);
    return (int)cudaGetLastError();
}

// forces of all wall subfaces of one block, accumulated into acc[12] (device)
static int launch_wall_forces(const Dims& d, const BlockDev& b, const std::vector<AdfbSubface>& subs, const double rp[3], double pRef,
                              double* acc, cudaStream_t s) {
    for (const AdfbSubface& sf : subs) {
        const bool viscWall = sf.bcType == ADFB_BC_NSWALL_ADIABATIC || sf.bcType == ADFB_BC_NSWALL_ISOTHERMAL;
        if (!viscWall && sf.bcType != ADFB_BC_EULERWALL) continue;
        FaceDev f = make_face(d, sf);
        const int dir = (sf.faceId - 1) / 2, isMin = (sf.faceId % 2) == 1;
        const int la = dir == 0 ? d.jl : d.il, lb = dir == 2 ? d.jl : d.kl;
        launch_kernel(K_MISC, true, 1, 256, 0, s, k_wall_forces, d, b, f, sf.iblank, dir, isMin, la, lb, viscWall ? 1 : 0, rp[0], rp[1], rp[2], pRef, acc);
    }
    return (int)cudaGetLastError();
}
