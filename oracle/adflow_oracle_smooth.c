/*
 * adflow_oracle_smooth.c -- CPU restatement of the boundary conditions and the
 * Runge-Kutta smoother of the ADflow hot path.  TEST INFRASTRUCTURE ONLY
 * (pinned bit-exact against oracle/_ref, see adflow_oracle.h).
 */
#include "orc_internal.h"

/* ------------------------------------------------------------------------ */
/* BC plane addressing == setBCPointers, src/utils/utils.F90:881-1174:
   plane 0 = 2nd halo, 1 = 1st halo, 2 = first interior, 3 = second interior;
   (a,b) are the two in-plane indices in the reference's order. */
typedef struct Face {
    long off[4];
    long sa, sb;
} Face;

static Face face_of(Dims d, int faceId) {
    Face f;
    switch (faceId) {
        case ADFB_IMIN: f.off[0] = 0; f.off[1] = 1; f.off[2] = 2; f.off[3] = 3; f.sa = d.sJ; f.sb = d.sK; break;
        case ADFB_IMAX: f.off[0] = d.ib; f.off[1] = d.ie; f.off[2] = d.il; f.off[3] = d.nx; f.sa = d.sJ; f.sb = d.sK; break;
        case ADFB_JMIN: f.off[0] = 0; f.off[1] = d.sJ; f.off[2] = 2 * d.sJ; f.off[3] = 3 * d.sJ; f.sa = 1; f.sb = d.sK; break;
        case ADFB_JMAX: f.off[0] = d.jb * d.sJ; f.off[1] = d.je * d.sJ; f.off[2] = d.jl * d.sJ; f.off[3] = d.ny * d.sJ; f.sa = 1; f.sb = d.sK; break;
        case ADFB_KMIN: f.off[0] = 0; f.off[1] = d.sK; f.off[2] = 2 * d.sK; f.off[3] = 3 * d.sK; f.sa = 1; f.sb = d.sJ; break;
        default: f.off[0] = d.kb * d.sK; f.off[1] = d.ke * d.sK; f.off[2] = d.kl * d.sK; f.off[3] = d.nz * d.sK; f.sa = 1; f.sb = d.sJ; break;
    }
    return f;
}
#define NRM(sf, a, b, m) ((sf)->norm[((a) - (sf)->icBeg) + na * (((b) - (sf)->jcBeg) + nb * (long)(m))])

/* computeEtot on one halo plane: src/solver/BCRoutines.F90:1816-1868 (cpConstant, no k) */
static void bc_etot(const OrcBlock* b, Dims d, double gam, long c) {
    double ovgm1 = one / (gam - one);
    W(c, IRHOE) = ovgm1 * b->p[c] + half * W(c, IRHO) * (W(c, IVX) * W(c, IVX) + W(c, IVY) * W(c, IVY) + W(c, IVZ) * W(c, IVZ));
}
/* extrapolate2ndHalo: src/solver/BCRoutines.F90:1870-1918 */
static void bc_extrap2(const OrcBlock* b, Dims d, const AdfbParams* prm, long c0, long c1, long c2) {
    const double factor = 0.5;
    W(c0, IRHO) = two * W(c1, IRHO) - W(c2, IRHO);
    W(c0, IRHO) = dmax(factor * W(c1, IRHO), W(c0, IRHO));
    W(c0, IVX) = two * W(c1, IVX) - W(c2, IVX);
    W(c0, IVY) = two * W(c1, IVY) - W(c2, IVY);
    W(c0, IVZ) = two * W(c1, IVZ) - W(c2, IVZ);
    b->p[c0] = dmax(factor * b->p[c1], two * b->p[c1] - b->p[c2]);
    if (prm->equations != ADFB_EULER) b->rlv[c0] = b->rlv[c1];
    if (prm->equations == ADFB_RANS) b->rev[c0] = b->rev[c1];
    bc_etot(b, d, prm->gammaInf, c0);
}

/* turbulence halo treatment of one subface: bcTurbTreatment + applyAllTurbBCThisBlock,
   src/turbulence/turbBCRoutines.F90:49-236,662-797 specialised to the scalar SA
   variable (bmt is 1x1): wall bmt=1 (:835-870), symm bmt=-1 (:614-660), far field
   bmt=-1 on outflow else bvt=wInf (:373-459); bcEddyWall/NoWall :238-372;
   turb2ndHalo :1132-1231. */
static void bc_turb_subface(const OrcBlock* b, const AdfbParams* prm, const AdfbSubface* sf, int secondHalo) {
    Dims d = dims_of(b);
    Face f = face_of(d, sf->faceId);
    long na = sf->icEnd - sf->icBeg + 1, nb = sf->jcEnd - sf->jcBeg + 1;
    for (int jb_ = sf->jcBeg; jb_ <= sf->jcEnd; jb_++) for (int ia = sf->icBeg; ia <= sf->icEnd; ia++) {
        long q = ia * f.sa + jb_ * f.sb;
        long c0 = f.off[0] + q, c1 = f.off[1] + q, c2 = f.off[2] + q;
        double bmt = zero, bvt = zero;
        int wall = sf->bcType == ADFB_BC_NSWALL_ADIABATIC || sf->bcType == ADFB_BC_NSWALL_ISOTHERMAL;
        if (wall) bmt = one;
        else if (sf->bcType == ADFB_BC_SYMM || sf->bcType == ADFB_BC_SYMMPOLAR) bmt = -one;   /* bcTurbSymm, turbBCRoutines.F90:765 */
        else if (sf->bcType == ADFB_BC_FARFIELD) {
            double dot = NRM(sf, ia, jb_, 0) * prm->wInf[IVX] + NRM(sf, ia, jb_, 1) * prm->wInf[IVY] +
                         NRM(sf, ia, jb_, 2) * prm->wInf[IVZ] - (sf->rface ? sf->rface[(ia - sf->icBeg) + na * (jb_ - sf->jcBeg)] : zero);
            if (dot > zero) bmt = -one; else bvt = prm->wInf[ITU1];
        } else if (sf->bcType == ADFB_BC_SUBSONIC_INFLOW || sf->bcType == ADFB_BC_SUPERSONIC_INFLOW) {
            /* bcTurbInflow, turbBCRoutines.F90:460-515 */
            long oo = (ia - sf->icBeg) + na * (jb_ - sf->jcBeg);
            bvt = two * (sf->turbInlet ? sf->turbInlet[oo] : zero);
            bmt = one;
        } else if (sf->bcType == ADFB_BC_SUBSONIC_OUTFLOW || sf->bcType == ADFB_BC_SUPERSONIC_OUTFLOW) bmt = -one; /* bcTurbOutflow */
        else if (sf->bcType == ADFB_BC_EULERWALL) bmt = -one; /* bcTurbSymm is used for Euler walls (:706) */
        else if (sf->bcType == ADFB_BC_EXTRAP) bmt = -one;     /* bcTurbOutflow: zero gradient (:564-613) */
        W(c1, ITU1) = bvt;
        W(c1, ITU1) = W(c1, ITU1) - bmt * W(c2, ITU1);
        if (wall) b->rev[c1] = -b->rev[c2]; else b->rev[c1] = b->rev[c2];
        if (secondHalo) { W(c0, ITU1) = W(c1, ITU1); b->rev[c0] = b->rev[c1]; }
    }
}

/* flow BC of one subface; phase selects symm 1st (1) / 2nd (2) halo, else the
   whole routine.  src/solver/BCRoutines.F90: bcSymm1stHalo :223, bcSymm2ndHalo :282,
   bcNSWallAdiabatic :489, bcFarfield :1282, bcEulerWall :1063, bcExtrap :1690. */
static void bc_flow_subface(const OrcBlock* b, const AdfbParams* prm, const AdfbSubface* sf, int secondHalo, int phase) {
    Dims d = dims_of(b);
    Face f = face_of(d, sf->faceId);
    long na = sf->icEnd - sf->icBeg + 1, nb = sf->jcEnd - sf->jcBeg + 1;
    int viscous = prm->equations != ADFB_EULER, eddy = prm->equations == ADFB_RANS;
    double gam = prm->gammaInf;
    for (int jb_ = sf->jcBeg; jb_ <= sf->jcEnd; jb_++) for (int ia = sf->icBeg; ia <= sf->icEnd; ia++) {
        long q = ia * f.sa + jb_ * f.sb;
        long c0 = f.off[0] + q, c1 = f.off[1] + q, c2 = f.off[2] + q, c3 = f.off[3] + q;
        double n1 = sf->norm ? NRM(sf, ia, jb_, 0) : zero, n2 = sf->norm ? NRM(sf, ia, jb_, 1) : zero,
               n3 = sf->norm ? NRM(sf, ia, jb_, 2) : zero;
        double rface = sf->rface ? sf->rface[(ia - sf->icBeg) + na * (jb_ - sf->jcBeg)] : zero;
        switch (sf->bcType) {
            case ADFB_BC_SYMM: {
                long ch = phase == 1 ? c1 : c0, ci = phase == 1 ? c2 : c3;
                double vn = two * (W(ci, IVX) * n1 + W(ci, IVY) * n2 + W(ci, IVZ) * n3);
                W(ch, IRHO) = W(ci, IRHO);
                W(ch, IVX) = W(ci, IVX) - vn * n1;
                W(ch, IVY) = W(ci, IVY) - vn * n2;
                W(ch, IVZ) = W(ci, IVZ) - vn * n3;
                W(ch, IRHOE) = W(ci, IRHOE);
                b->p[ch] = b->p[ci];
                if (viscous) b->rlv[ch] = b->rlv[ci];
                if (eddy) b->rev[ch] = b->rev[ci];
                break;
            }
            case ADFB_BC_SYMMPOLAR: {  /* bcSymmPolar1stHalo / 2ndHalo, BCRoutines.F90:332-486 */
                long ch = phase == 1 ? c1 : c0, ci = phase == 1 ? c2 : c3;
                /* xx(i+1,j+1,:) - xx(i,j,:): diagonal of the (collapsed) boundary face, nodes (ia,jb) and (ia-1,jb-1) */
                int isMin = sf->faceId == ADFB_IMIN || sf->faceId == ADFB_JMIN || sf->faceId == ADFB_KMIN;
                long xo = isMin ? f.off[1] : f.off[2];
                long nA = xo + ia * f.sa + jb_ * f.sb, nB = xo + (ia - 1) * f.sa + (jb_ - 1) * f.sb;
                double nnx = X(nA, 0) - X(nB, 0), nny = X(nA, 1) - X(nB, 1), nnz = X(nA, 2) - X(nB, 2);
                double tmp = one / sqrt(nnx * nnx + nny * nny + nnz * nnz);
                nnx = nnx * tmp; nny = nny * tmp; nnz = nnz * tmp;
                tmp = two * (W(ci, IVX) * nnx + W(ci, IVY) * nny + W(ci, IVZ) * nnz);
                double vtx = tmp * nnx, vty = tmp * nny, vtz = tmp * nnz;
                W(ch, IRHO) = W(ci, IRHO);
                W(ch, IVX) = vtx - W(ci, IVX);
                W(ch, IVY) = vty - W(ci, IVY);
                W(ch, IVZ) = vtz - W(ci, IVZ);
                W(ch, IRHOE) = W(ci, IRHOE);
                b->p[ch] = b->p[ci];
                if (viscous) b->rlv[ch] = b->rlv[ci];
                if (eddy) b->rev[ch] = b->rev[ci];
                break;
            }
            case ADFB_BC_NSWALL_ADIABATIC: {
                double us1 = zero, us2 = zero, us3 = zero;
                if (sf->uSlip) {
                    long o = (ia - sf->icBeg) + na * (jb_ - sf->jcBeg);
                    us1 = sf->uSlip[o]; us2 = sf->uSlip[o + na * nb]; us3 = sf->uSlip[o + 2 * na * nb];
                }
                W(c1, IRHO) = W(c2, IRHO);
                W(c1, IVX) = -W(c2, IVX) + two * us1;
                W(c1, IVY) = -W(c2, IVY) + two * us2;
                W(c1, IVZ) = -W(c2, IVZ) + two * us3;
                b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = -b->rev[c2];
                if (prm->wallBCConstantPressure) {
                    b->p[c1] = b->p[c2] - four * third * zero;
                } else {
                    b->p[c1] = 2 * b->p[c2] - b->p[c3];
                    if (b->p[c1] <= zero) b->p[c1] = b->p[c2];
                }
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            case ADFB_BC_NSWALL_ISOTHERMAL: { /* bcNSWallIsoThermal, BCRoutines.F90:579-691 */
                double us1 = zero, us2 = zero, us3 = zero;
                long o = (ia - sf->icBeg) + na * (jb_ - sf->jcBeg);
                if (sf->uSlip) { us1 = sf->uSlip[o]; us2 = sf->uSlip[o + na * nb]; us3 = sf->uSlip[o + 2 * na * nb]; }
                double tw = sf->TNSWall[o];
                double t2 = b->p[c2] / (prm->RGas * W(c2, IRHO));
                double t1 = two * tw - t2;
                t1 = dmax(half * tw, t1);
                t1 = dmin(two * tw, t1);
                if (prm->wallBCConstantPressure) {
                    b->p[c1] = b->p[c2] - four * third * zero;
                } else {
                    b->p[c1] = 2 * b->p[c2] - b->p[c3];
                    if (b->p[c1] <= zero) b->p[c1] = b->p[c2];
                }
                W(c1, IRHO) = b->p[c1] / (prm->RGas * t1);
                W(c1, IVX) = -W(c2, IVX) + two * us1;
                W(c1, IVY) = -W(c2, IVY) + two * us2;
                W(c1, IVZ) = -W(c2, IVZ) + two * us3;
                b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = -b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            case ADFB_BC_SUBSONIC_OUTFLOW: { /* bcSubsonicOutflow, BCRoutines.F90:693-802 */
                long o = (ia - sf->icBeg) + na * (jb_ - sf->jcBeg);
                double pExit = sf->ps[o];
                double ovg = one / gam, ovgm1 = one / (gam - one);
                double pInt = b->p[c2];
                double r = one / W(c2, IRHO);
                double a2 = gam * pInt * r;
                double a = sqrt(a2);
                double ue = W(c2, IVX), ve = W(c2, IVY), we = W(c2, IVZ);
                double qne = ue * n1 + ve * n2 + we * n3;
                double ss = pInt * pow(r, gam);
                double ac = qne + two * a * ovgm1;
                W(c1, IRHO) = pow(pExit / ss, ovg);
                b->p[c1] = pExit;
                a = sqrt(gam * pExit / W(c1, IRHO));
                double qnh = ac - two * a * ovgm1;
                W(c1, IVX) = ue + (qnh - qne) * n1;
                W(c1, IVY) = ve + (qnh - qne) * n2;
                W(c1, IVZ) = we + (qnh - qne) * n3;
                if (viscous) b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            case ADFB_BC_SUBSONIC_INFLOW: { /* bcSubsonicInflow, BCRoutines.F90:804-1061, cpConstant */
                long o = (ia - sf->icBeg) + na * (jb_ - sf->jcBeg);
                double govgm1 = gam / (gam - one);
                double gm1 = gam - one, ovgm1 = one / gm1;
                double r = one / W(c2, IRHO);
                double a2 = gam * b->p[c2] * r;
                double beta = W(c2, IVX) * n1 + W(c2, IVY) * n2 + W(c2, IVZ) * n3 + two * ovgm1 * sqrt(a2);
                if (sf->subsonicInletTreatment == 1) { /* totalConditions */
                    double ptot = sf->ptInlet[o], ttot = sf->ttInlet[o], htot = sf->htInlet[o];
                    double ssx = sf->flowXdirInlet[o], ssy = sf->flowYdirInlet[o], ssz = sf->flowZdirInlet[o];
                    double scaleFact = one;
                    if (prm->hScalingInlet) scaleFact = sqrt(htot / (r * (W(c2, IRHOE) + b->p[c2])));
                    beta = beta * scaleFact;
                    double q2 = W(c2, IVX) * W(c2, IVX) + W(c2, IVY) * W(c2, IVY) + W(c2, IVZ) * W(c2, IVZ);
                    double a2tot = gm1 * (htot - r * (W(c2, IRHOE) + b->p[c2]) + half * q2) + a2;
                    double alpha = n1 * ssx + n2 * ssy + n3 * ssz;
                    double aa2 = half * gm1 * alpha * alpha + one;
                    double bb = -gm1 * alpha * beta;
                    double cc = half * gm1 * beta * beta - two * ovgm1 * a2tot;
                    double dd = bb * bb - four * aa2 * cc;
                    dd = sqrt(dmax(zero, dd));
                    double q = (-bb + dd) / (two * aa2);
                    q = dmax(zero, q);
                    q2 = q * q;
                    a2 = a2tot - half * gm1 * q2;
                    double m2 = q2 / a2;
                    m2 = dmin(one, m2);
                    q2 = m2 * a2;
                    q = sqrt(q2);
                    a2 = a2tot - half * gm1 * q2;
                    W(c1, IVX) = q * ssx; W(c1, IVY) = q * ssy; W(c1, IVZ) = q * ssz;
                    double ts = a2 / (gam * prm->RGas);
                    double ratio = pow(ts / ttot, govgm1);
                    b->p[c1] = ptot * ratio;
                    W(c1, IRHO) = (ptot * ratio) / (prm->RGas * ts);
                } else { /* massFlow */
                    double rho = sf->rho[o], velx = sf->velx[o], vely = sf->vely[o], velz = sf->velz[o];
                    a2 = half * gm1 * (beta - velx * n1 - vely * n2 - velz * n3);
                    a2 = dmax(zero, a2);
                    a2 = a2 * a2;
                    b->p[c1] = rho * a2 / gam;
                    W(c1, IRHO) = rho; W(c1, IVX) = velx; W(c1, IVY) = vely; W(c1, IVZ) = velz;
                }
                if (viscous) b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            case ADFB_BC_SUPERSONIC_INFLOW: { /* bcSupersonicInflow, BCRoutines.F90:1411-1477 */
                long o = (ia - sf->icBeg) + na * (jb_ - sf->jcBeg);
                W(c1, IRHO) = sf->rho[o]; W(c1, IVX) = sf->velx[o]; W(c1, IVY) = sf->vely[o]; W(c1, IVZ) = sf->velz[o];
                b->p[c1] = sf->ps[o];
                if (viscous) b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) {
                    W(c0, IRHO) = sf->rho[o]; W(c0, IVX) = sf->velx[o]; W(c0, IVY) = sf->vely[o]; W(c0, IVZ) = sf->velz[o];
                    b->p[c0] = sf->ps[o];
                    if (viscous) b->rlv[c0] = b->rlv[c1];
                    if (eddy) b->rev[c0] = b->rev[c1];
                    bc_etot(b, d, gam, c0);
                }
                break;
            }
            case ADFB_BC_EXTRAP:
            case ADFB_BC_SUPERSONIC_OUTFLOW: { /* bcExtrap, BCRoutines.F90:1479-1570 */
                double fw2 = two, fw3 = -one, factor = half;
                if (sf->bcType == ADFB_BC_SUPERSONIC_OUTFLOW && !prm->outflowLinearExtrapol) { fw2 = one; fw3 = zero; }
                W(c1, IRHO) = fw2 * W(c2, IRHO) + fw3 * W(c3, IRHO);
                W(c1, IRHO) = dmax(factor * W(c2, IRHO), W(c1, IRHO));
                W(c1, IVX) = fw2 * W(c2, IVX) + fw3 * W(c3, IVX);
                W(c1, IVY) = fw2 * W(c2, IVY) + fw3 * W(c3, IVY);
                W(c1, IVZ) = fw2 * W(c2, IVZ) + fw3 * W(c3, IVZ);
                b->p[c1] = fw2 * b->p[c2] + fw3 * b->p[c3];
                b->p[c1] = dmax(factor * b->p[c2], b->p[c1]);
                if (viscous) b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            case ADFB_BC_FARFIELD: {
                double gm1 = gam - one, ovgm1 = one / gm1;
                double r0 = one / prm->wInf[IRHO], u0 = prm->wInf[IVX], v0 = prm->wInf[IVY], w0 = prm->wInf[IVZ];
                double c0s = sqrt(gam * prm->pInfCorr * r0);
                double s0 = pow(prm->wInf[IRHO], gam) / prm->pInfCorr;
                double qn0 = u0 * n1 + v0 * n2 + w0 * n3;
                double vn0 = qn0 - rface;
                double re = one / W(c2, IRHO), ue = W(c2, IVX), ve = W(c2, IVY), we = W(c2, IVZ);
                double qne = ue * n1 + ve * n2 + we * n3;
                double ce = sqrt(gam * b->p[c2] * re);
                double ac1, ac2;
                if (vn0 > -c0s) ac1 = qne + two * ovgm1 * ce; else ac1 = qn0 + two * ovgm1 * c0s;
                if (vn0 > c0s) ac2 = qne - two * ovgm1 * ce; else ac2 = qn0 - two * ovgm1 * c0s;
                double qnf = half * (ac1 + ac2);
                double cf = fourth * (ac1 - ac2) * gm1;
                double uf, vf, wf, sfv;
                if (vn0 > zero) {
                    uf = ue + (qnf - qne) * n1; vf = ve + (qnf - qne) * n2; wf = we + (qnf - qne) * n3;
                    sfv = pow(W(c2, IRHO), gam) / b->p[c2];
                } else {
                    uf = u0 + (qnf - qn0) * n1; vf = v0 + (qnf - qn0) * n2; wf = w0 + (qnf - qn0) * n3;
                    sfv = s0;
                }
                double cc = cf * cf / gam;
                W(c1, IRHO) = pow(sfv * cc, ovgm1);
                W(c1, IVX) = uf; W(c1, IVY) = vf; W(c1, IVZ) = wf;
                b->p[c1] = W(c1, IRHO) * cc;
                if (viscous) b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            case ADFB_BC_EULERWALL: {
                /* eulerWallBCTreatment: linear pressure extrapolation (pyADflow default) or
                   constant pressure; the normal-momentum variant is not restated */
                double grad = prm->reserved ? zero : b->p[c3] - b->p[c2];
                b->p[c1] = fdim_(b->p[c2], grad);
                double vn = two * (rface - W(c2, IVX) * n1 - W(c2, IVY) * n2 - W(c2, IVZ) * n3);
                W(c1, IRHO) = W(c2, IRHO);
                W(c1, IVX) = W(c2, IVX) + vn * n1;
                W(c1, IVY) = W(c2, IVY) + vn * n2;
                W(c1, IVZ) = W(c2, IVZ) + vn * n3;
                if (viscous) b->rlv[c1] = b->rlv[c2];
                if (eddy) b->rev[c1] = b->rev[c2];
                bc_etot(b, d, gam, c1);
                if (secondHalo) bc_extrap2(b, d, prm, c0, c1, c2);
                break;
            }
            default: break;
        }
    }
}

/* applyAllTurbBCThisBlock order: subfaces in nBocos order */
void orc_apply_turb_bc(const OrcBlock* b, const AdfbParams* prm, int nSub, const AdfbSubface* sf, int secondHalo) {
    if (prm->equations != ADFB_RANS) return;
    for (int n = 0; n < nSub; n++) bc_turb_subface(b, prm, &sf[n], secondHalo);
}
/* applyAllBC_block order, src/solver/BCRoutines.F90:81-216: symm 1st halo, symm 2nd
   halo, (polar), adiabatic walls, isothermal walls, far field, (outflow, inflow),
   extrapolation, Euler walls, (supersonic inflow) */
void orc_apply_flow_bc(const OrcBlock* b, const AdfbParams* prm0, int nSub, const AdfbSubface* sf, int secondHalo) {
    int n;
    /* coarse levels: constant pressure at viscous and inviscid walls, BCRoutines.F90:550,642,1100 */
    AdfbParams prmL = *prm0;
    if (b->level > 1) { prmL.wallBCConstantPressure = 1; prmL.reserved = 1; }
    const AdfbParams* prm = &prmL;
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SYMM) bc_flow_subface(b, prm, &sf[n], secondHalo, 1);
    if (secondHalo) for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SYMM) bc_flow_subface(b, prm, &sf[n], secondHalo, 2);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SYMMPOLAR) bc_flow_subface(b, prm, &sf[n], secondHalo, 1);
    if (secondHalo) for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SYMMPOLAR) bc_flow_subface(b, prm, &sf[n], secondHalo, 2);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_NSWALL_ADIABATIC) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_NSWALL_ISOTHERMAL) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_FARFIELD) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SUBSONIC_OUTFLOW) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SUBSONIC_INFLOW) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++)
        if (sf[n].bcType == ADFB_BC_EXTRAP || sf[n].bcType == ADFB_BC_SUPERSONIC_OUTFLOW) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_EULERWALL) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
    for (n = 0; n < nSub; n++) if (sf[n].bcType == ADFB_BC_SUPERSONIC_INFLOW) bc_flow_subface(b, prm, &sf[n], secondHalo, 0);
}

/* ------------------------------------------------------------------------ */
/* residualAveraging: src/solver/residuals.F90:1785-2080 (fine level: cfl) */
static double ra_rfl(const OrcBlock* b, Dims d, long c, double plim) {
    const double* p = b->p;
    double dpi = fabs(p[c + 1] - two * p[c] + p[c - 1]) / (p[c + 1] + two * p[c] + p[c - 1] + plim);
    double dpj = fabs(p[c + d.sJ] - two * p[c] + p[c - d.sJ]) / (p[c + d.sJ] + two * p[c] + p[c - d.sJ] + plim);
    double dpk = fabs(p[c + d.sK] - two * p[c] + p[c - d.sK]) / (p[c + d.sK] + two * p[c] + p[c - d.sK] + plim);
    return one / (one + 2.0 * (dpi + dpj + dpk));
}
/* one direction: lines of n owned cells with stride sd; other two owned ranges looped */
static void ra_dir(const OrcBlock* b, const AdfbParams* prm, Dims d, long sd, int n, long s1, int n1, long s2, int n2) {
    if (n <= 1) return;
    double rfl0 = half * prm->cfl / prm->cflLimit, plim = 0.001 * prm->pInfCorr;
    int l = n + 1; /* il-equivalent along the line: owned 2..l */
    double* epz = (double*)malloc(sizeof(double) * (l + 2));
    double* dd = (double*)malloc(sizeof(double) * (l + 2));
    double* t = (double*)malloc(sizeof(double) * (l + 2));
    for (int q2 = 2; q2 <= n2 + 1; q2++) for (int q1 = 2; q1 <= n1 + 1; q1++) {
        long base = q1 * s1 + q2 * s2;
        for (int i = 2; i <= n; i++) {
            long c = base + i * sd;
            double r = rfl0 * (ra_rfl(b, d, c, plim) + ra_rfl(b, d, c + sd, plim));
            epz[i] = fourth * prm->smoop * fdim_(r * r, one) * dmax((double)b->iblank[c], zero);
        }
        epz[1] = zero; epz[l] = zero; dd[1] = zero;
        for (int i = 2; i <= l; i++) {
            t[i] = one / (one + epz[i] + epz[i - 1] - epz[i - 1] * dd[i - 1]);
            dd[i] = t[i] * epz[i];
        }
        for (int i = 2; i <= l; i++) {
            long c = base + i * sd;
            for (int m = 0; m < 5; m++) DW(c, m) = t[i] * (DW(c, m) + epz[i - 1] * DW(c - sd, m));
        }
        for (int i = n; i >= 2; i--) {
            long c = base + i * sd;
            for (int m = 0; m < 5; m++) DW(c, m) = DW(c, m) + dd[i] * DW(c + sd, m);
        }
    }
    free(epz); free(dd); free(t);
}
void orc_residual_averaging(const OrcBlock* b, const AdfbParams* prm) {
    Dims d = dims_of(b);
    ra_dir(b, prm, d, d.sI, d.nx, d.sJ, d.ny, d.sK, d.nz);
    ra_dir(b, prm, d, d.sJ, d.ny, d.sI, d.nx, d.sK, d.nz);
    ra_dir(b, prm, d, d.sK, d.nz, d.sI, d.nx, d.sJ, d.ny);
}

/* ------------------------------------------------------------------------ */
/* block-path mean-flow residual used by the smoothers:
   initres (fine grid steady: dw = 0, src/solver/residuals.F90:427-497) +
   residual_block (:4-346) with rFil = cdisRK(rkStage+1) for the RK smoother.
   Radii are NOT recomputed (timeStep is a separate call in executeMGCycle). */
void orc_residual_block(const OrcBlock* b, const AdfbParams* prm, double rFil) {
    if (b->level > 1) { orc_residual_block_coarse(b, prm, rFil, 1); return; }  /* initRes: dw = wr, 1st-order dissipation */
    Dims d = dims_of(b);
    int viscous = prm->equations != ADFB_EULER;
    memset(b->dw, 0, sizeof(double) * 5 * d.N);
    orc_central_flux(b, prm);
    if (fabs(rFil) >= thresholdReal) {
        /* orc_diss_scalar recomputes ss/dss and scales fw by (1-rFil) like fluxes.F90:1193 */
        if (prm->spaceDiscr == ADFB_DISS_SCALAR) orc_diss_scalar(b, prm, rFil);
        else if (prm->spaceDiscr == ADFB_DISS_MATRIX) orc_diss_matrix(b, prm, rFil);
        else orc_upwind_flux(b, prm, rFil);
        if (viscous) {
            orc_speed_of_sound(b, prm);
            orc_nodal_gradients(b);
            orc_viscous_flux(b, prm, rFil);
        }
    }
    orc_sum_dw_fw(b);
}

/* executeRkStage: src/solver/smoothers.F90:90-382 (steady, fine level, no precond);
   BCs and halo exchange are the caller's (single block: BCs only). */
void orc_rk_stage(const OrcBlock* b, const AdfbParams* prm0, int rkStage, int nSub, const AdfbSubface* sf) {
    Dims d = dims_of(b);
    /* currentCfl = cflCoarse unless currentLevel == 1; secondHalo only on the ground level (smoothers.F90:131-140) */
    AdfbParams prmL = *prm0;
    if (b->level > 1) prmL.cfl = prm0->cflCoarse;
    const AdfbParams* prm = &prmL;
    double tmp = prm->cfl * prm->etaRK[rkStage - 1];
    int smooth = prm->resAveraging == 1 || (prm->resAveraging == 2 && (rkStage % 2) == 1);
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double dt = tmp * b->dtl[c];
        for (int l = 0; l < 5; l++) DW(c, l) = DW(c, l) * dt;
    }
    if (smooth) orc_residual_averaging(b, prm);
    double gm1 = prm->gammaInf - one;
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double ovr = one / W(c, IRHO);
        double v2 = W(c, IVX) * W(c, IVX) + W(c, IVY) * W(c, IVY) + W(c, IVZ) * W(c, IVZ);
        double factK = zero;
        double dp = (ovr * b->p[c] + factK - gm1 * (ovr * W(c, IRHOE) - v2)) * DW(c, IRHO) +
                    gm1 * (DW(c, IRHOE) - W(c, IVX) * DW(c, IMX) - W(c, IVY) * DW(c, IMY) - W(c, IVZ) * DW(c, IMZ));
        const double* wn = b->wn;
        W(c, IRHO) = wn[c] - DW(c, IRHO);
        W(c, IRHO) = dmax(W(c, IRHO), 1.e-4 * prm->rhoInf);
        double ru = wn[c] * wn[d.N + c] - DW(c, IMX);
        double rv = wn[c] * wn[2 * d.N + c] - DW(c, IMY);
        double rw = wn[c] * wn[3 * d.N + c] - DW(c, IMZ);
        ovr = one / W(c, IRHO);
        W(c, IVX) = ovr * ru; W(c, IVY) = ovr * rv; W(c, IVZ) = ovr * rw;
        b->p[c] = b->pn[c] - dp;
        b->p[c] = dmax(b->p[c], 1.e-4 * prm->pInfCorr);
    }
    orc_etot(b, prm, 2, d.il, 2, d.jl, 2, d.kl);
    orc_lam_viscosity(b, prm, 0);
    orc_eddy_viscosity(b, prm, 0);
    orc_apply_flow_bc(b, prm, nSub, sf, b->level > 1 ? 0 : 1);
}

/* RungeKuttaSmoother: src/solver/smoothers.F90:4-86.  On entry residual (rFil =
   cdisRK(1)) and dtl are assumed computed, like the reference. */
void orc_rk_smoother(const OrcBlock* b, const AdfbParams* prm, int nSub, const AdfbSubface* sf) {
    Dims d = dims_of(b);
    for (int l = 0; l < 5; l++) memcpy(b->wn + (long)l * d.N, b->w + (long)l * d.N, sizeof(double) * d.N);
    memcpy(b->pn, b->p, sizeof(double) * d.N);
    for (int st = 1; st <= prm->nRKStages - 1; st++) {
        orc_rk_stage(b, prm, st, nSub, sf);
        orc_residual_block(b, prm, prm->cdisRK[st]);
    }
    orc_rk_stage(b, prm, prm->nRKStages, nSub, sf);
}

/* ------------------------------------------------------------------------ */
/* tridiagsolve: src/solver/residuals.F90:1750-1783 (5 systems, rows 2..nn) */
static void tridiagsolve(double* bb, double* cc, double* dd, double* ff, int nn, int ld) {
    for (int n = 0; n < 5; n++) {
        double* b = bb + n * ld; double* c = cc + n * ld; double* d = dd + n * ld; double* f = ff + n * ld;
        int m = 2;
        double d0 = 1. / c[m];
        d[m] = d[m] * d0;
        f[m] = f[m] * d0;
        for (m = 3; m <= nn; m++) {
            double d2 = b[m];
            d0 = 1. / (c[m] - d2 * d[m - 1]);
            f[m] = (f[m] - d2 * f[m - 1]) * d0;
            d[m] = d[m] * d0;
        }
        for (m = nn - 1; m >= 2; m--) f[m] = f[m] - d[m] * f[m + 1];
    }
}

/* one implicit sweep of computedwDADI along direction `sd` (j :1333-1405, i :1470-1538,
   k :1605-1674).  s = face normals of the sweep direction; s2 = the array used in the
   metric average of eps2: the k sweep uses sj for the lower face (reference quirk,
   residuals.F90:1625-1627).  qq/cc are the scratch slots of the direction. */
static void dadi_sweep(const OrcBlock* b, const AdfbParams* prm, Dims d, long sd, int nl, const double* s, const double* slow,
                       const double* qq, const double* cc, const double* dual_dt, long s1, int n1, long s2, int n2) {
    const double epsval = 0.08, fac = 1.05;
    double cInf2 = prm->gammaInf * prm->pInf / prm->rhoInf;
    int viscous = prm->equations != ADFB_EULER, eddy = prm->equations == ADFB_RANS;
    int l = nl + 1, e = nl + 2; /* il, ie along the line */
    if (l <= 2) return;
    int ld = e + 2;
    double* bb = (double*)calloc(5 * ld, sizeof(double)); double* ccv = (double*)calloc(5 * ld, sizeof(double));
    double* dd = (double*)calloc(5 * ld, sizeof(double)); double* ff = (double*)calloc(5 * ld, sizeof(double));
    double* metterm = (double*)calloc(ld, sizeof(double));
    for (int q2 = 2; q2 <= n2 + 1; q2++) for (int q1 = 2; q1 <= n1 + 1; q1++) {
        long base = q1 * s1 + q2 * s2;
        for (int m = 1; m <= l; m++) {
            long c = base + m * sd;
            double mut = zero;
            if (viscous) mut = b->rlv[c] + b->rlv[c + sd];
            if (eddy) mut = mut + b->rev[c] + b->rev[c + sd];
            double volfact = one / (b->vol[c] + b->vol[c + sd]);
            double mt = s[c] * s[c] + s[d.N + c] * s[d.N + c] + s[2 * d.N + c] * s[2 * d.N + c];
            metterm[m] = mt * mut * volfact;
        }
        for (int m = 2; m <= l; m++) {
            long c = base + m * sd;
            double viscTerm1 = metterm[m] / b->vol[c] / W(c, IRHO);
            double viscTerm3 = metterm[m - 1] / b->vol[c] / W(c, IRHO);
            double viscTerm2 = viscTerm1 + viscTerm3;
            double volhalf = half / b->vol[c];
            double r1 = volhalf * (s[c] + slow[c - sd]);
            double r2 = volhalf * (s[d.N + c] + slow[d.N + c - sd]);
            double r3 = volhalf * (s[2 * d.N + c] + slow[2 * d.N + c - sd]);
            double mt = r1 * r1 + r2 * r2 + r3 * r3;
            double eps2 = epsval * epsval * cInf2 * mt;
            double q = qq[c], cs = cc[c];
            double dP[5], dM[5];
            dP[0] = half * (q + fac * sqrt(q * q + eps2)); dP[1] = dP[0]; dP[2] = dP[0];
            dP[3] = half * (q + cs + fac * sqrt((q + cs) * (q + cs) + eps2));
            dP[4] = half * (q - cs + fac * sqrt((q - cs) * (q - cs) + eps2));
            dM[0] = half * (q - fac * sqrt(q * q + eps2)); dM[1] = dM[0]; dM[2] = dM[0];
            dM[3] = half * (q + cs - fac * sqrt((q + cs) * (q + cs) + eps2));
            dM[4] = half * (q - cs - fac * sqrt((q - cs) * (q - cs) + eps2));
            for (int n = 0; n < 5; n++) {
                bb[n * ld + m + 1] = -viscTerm1 - dP[n];
                dd[n * ld + m - 1] = -viscTerm3 + dM[n];
                ccv[n * ld + m] = viscTerm2 + dP[n] - dM[n];
            }
        }
        for (int n = 0; n < 5; n++) {
            bb[n * ld + e] = zero;
            dd[n * ld + 1] = zero;
            dd[n * ld + l] = zero; /* never set by the reference (read but unused) */
            for (int m = 2; m <= l; m++) {
                long c = base + m * sd;
                double rb = dmax((double)b->iblank[c], zero);
                bb[n * ld + m] = bb[n * ld + m] * dual_dt[c] * rb;
                dd[n * ld + m] = dd[n * ld + m] * dual_dt[c] * rb;
                ccv[n * ld + m] = one + ccv[n * ld + m] * dual_dt[c] * rb + zero + zero;
                ff[n * ld + m] = DW(c, n);
            }
        }
        tridiagsolve(bb, ccv, dd, ff, l, ld);
        for (int n = 0; n < 5; n++) for (int m = 2; m <= l; m++) DW(base + m * sd, n) = ff[n * ld + m];
    }
    free(bb); free(ccv); free(dd); free(ff); free(metterm);
}

/* rotation between two characteristic bases (residuals.F90:1407-1448 with (ri,rj), :1543-1583 with (ri,rk)) */
static void dadi_rotate(const OrcBlock* b, Dims d, const double* sa, long sda, const double* sb, long sdb, int second) {
    const double sqrt2inv = one / sqrt(two);
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double a_[3], b_[3];
        for (int m = 0; m < 3; m++) { a_[m] = half * (sa[m * d.N + c] + sa[m * d.N + c - sda]); b_[m] = half * (sb[m * d.N + c] + sb[m * d.N + c - sdb]); }
        double ra = sqrt(a_[0] * a_[0] + a_[1] * a_[1] + a_[2] * a_[2]);
        a_[0] /= ra; a_[1] /= ra; a_[2] /= ra;
        double rb = sqrt(b_[0] * b_[0] + b_[1] * b_[1] + b_[2] * b_[2]);
        b_[0] /= rb; b_[1] /= rb; b_[2] /= rb;
        double dw1 = DW(c, 0), dw2 = DW(c, 1), dw3 = DW(c, 2), dw4 = DW(c, 3), dw5 = DW(c, 4);
        double a1, a2, a3, a4;
        const double *ri = a_, *rx = b_;
        a1 = ri[0] * rx[0] + ri[1] * rx[1] + ri[2] * rx[2];
        if (!second) { /* (ri, rj) */
            a2 = ri[0] * rx[1] - rx[0] * ri[1];
            a3 = ri[2] * rx[1] - rx[2] * ri[1];
            a4 = ri[0] * rx[2] - rx[0] * ri[2];
        } else {       /* (ri, rk): a2 = rk1*ri2 - ri1*rk2 ... */
            a2 = rx[0] * ri[1] - ri[0] * rx[1];
            a3 = rx[2] * ri[1] - ri[2] * rx[1];
            a4 = rx[0] * ri[2] - ri[0] * rx[2];
        }
        double a5 = (dw4 - dw5) * sqrt2inv;
        double a6 = (dw4 + dw5) * half;
        double a7 = (a3 * dw1 + a4 * dw2 - a2 * dw3 - a5 * a1) * sqrt2inv;
        DW(c, 0) = a1 * dw1 + a2 * dw2 + a4 * dw3 + a5 * a3;
        DW(c, 1) = -a2 * dw1 + a1 * dw2 - a3 * dw3 + a5 * a4;
        DW(c, 2) = -a4 * dw1 + a3 * dw2 + a1 * dw3 - a5 * a2;
        DW(c, 3) = -a7 + a6;
        DW(c, 4) = a7 + a6;
    }
}

/* computedwDADI: src/solver/residuals.F90:1062-1748 (steady; spectral_* are multiplied by
   zero in the reference (:1269-1271) and therefore omitted) */
void orc_compute_dw_dadi(const OrcBlock* b, const AdfbParams* prm) {
    Dims d = dims_of(b);
    double* qq_i = b->scratch, *qq_j = b->scratch + d.N, *qq_k = b->scratch + 2 * d.N;
    double* cc_i = b->scratch + 3 * d.N, *cc_j = b->scratch + 4 * d.N, *cc_k = b->scratch + 5 * d.N;
    double* dual_dt = b->scratch + 9 * d.N;
    const double sqrt2 = sqrt(two);
    double gam = prm->gammaInf;
    const double *si = b->si, *sj = b->sj, *sk = b->sk;
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        dual_dt[c] = prm->cfl * b->dtl[c] * b->vol[c];
    }
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double volhalf = half / b->vol[c];
        double cijk = sqrt(gam * b->p[c] / W(c, IRHO));
        double ri1 = volhalf * (si[c] + si[c - 1]), ri2 = volhalf * (si[d.N + c] + si[d.N + c - 1]), ri3 = volhalf * (si[2 * d.N + c] + si[2 * d.N + c - 1]);
        double rj1 = volhalf * (sj[c] + sj[c - d.sJ]), rj2 = volhalf * (sj[d.N + c] + sj[d.N + c - d.sJ]), rj3 = volhalf * (sj[2 * d.N + c] + sj[2 * d.N + c - d.sJ]);
        double rk1 = volhalf * (sk[c] + sk[c - d.sK]), rk2 = volhalf * (sk[d.N + c] + sk[d.N + c - d.sK]), rk3 = volhalf * (sk[2 * d.N + c] + sk[2 * d.N + c - d.sK]);
        qq_i[c] = ri1 * W(c, IVX) + ri2 * W(c, IVY) + ri3 * W(c, IVZ) - zero;
        qq_j[c] = rj1 * W(c, IVX) + rj2 * W(c, IVY) + rj3 * W(c, IVZ) - zero;
        qq_k[c] = rk1 * W(c, IVX) + rk2 * W(c, IVY) + rk3 * W(c, IVZ) - zero;
        cc_i[c] = cijk * sqrt(ri1 * ri1 + ri2 * ri2 + ri3 * ri3);
        cc_j[c] = cijk * sqrt(rj1 * rj1 + rj2 * rj2 + rj3 * rj3);
        cc_k[c] = cijk * sqrt(rk1 * rk1 + rk2 * rk2 + rk3 * rk3);
    }
    /* T_eta^-1: conservative -> characteristic variables of the j direction (:1277-1327) */
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double gm1 = gam - one;
        double cijk = sqrt(gam * b->p[c] / W(c, IRHO));
        double c2inv = one / (cijk * cijk);
        double xfact = two * cijk;
        double alphinv = sqrt2 * cijk / W(c, IRHO);
        double uvel = W(c, IVX), vvel = W(c, IVY), wvel = W(c, IVZ);
        double uvw = half * (uvel * uvel + vvel * vvel + wvel * wvel);
        double rj1 = half * (sj[c] + sj[c - d.sJ]), rj2 = half * (sj[d.N + c] + sj[d.N + c - d.sJ]), rj3 = half * (sj[2 * d.N + c] + sj[2 * d.N + c - d.sJ]);
        double rj = sqrt(rj1 * rj1 + rj2 * rj2 + rj3 * rj3);
        double uu = uvel * rj1 + vvel * rj2 + wvel * rj3;
        rj1 = rj1 / rj; rj2 = rj2 / rj; rj3 = rj3 / rj;
        double dw1 = DW(c, 0), dw2 = DW(c, 1), dw3 = DW(c, 2), dw4 = DW(c, 3), dw5 = DW(c, 4);
        double a1 = dw2 * uvel + dw3 * vvel + dw4 * wvel - dw5;
        a1 = a1 * gm1 * c2inv + dw1 * (one - uvw * gm1 * c2inv);
        double a2 = (rj2 * wvel - rj3 * vvel) * dw1 + rj3 * dw3 - rj2 * dw4;
        double a3 = (rj3 * uvel - rj1 * wvel) * dw1 + rj1 * dw4 - rj3 * dw2;
        double a4 = (rj1 * vvel - rj2 * uvel) * dw1 + rj2 * dw2 - rj1 * dw3;
        double a5 = uvw * dw1 - uvel * dw2 - vvel * dw3 - wvel * dw4 + dw5;
        a5 = a5 * gm1 * c2inv;
        double a6 = uu * dw1 / rj - rj1 * dw2 - rj2 * dw3 - rj3 * dw4;
        DW(c, 0) = a1 * rj1 + a2 / W(c, IRHO);
        DW(c, 1) = a1 * rj2 + a3 / W(c, IRHO);
        DW(c, 2) = a1 * rj3 + a4 / W(c, IRHO);
        DW(c, 3) = (half * a5 - a6 / xfact) * alphinv;
        DW(c, 4) = (half * a5 + a6 / xfact) * alphinv;
    }
    dadi_sweep(b, prm, d, d.sJ, d.ny, sj, sj, qq_j, cc_j, dual_dt, d.sI, d.nx, d.sK, d.nz);
    dadi_rotate(b, d, si, d.sI, sj, d.sJ, 0);
    dadi_sweep(b, prm, d, d.sI, d.nx, si, si, qq_i, cc_i, dual_dt, d.sJ, d.ny, d.sK, d.nz);
    dadi_rotate(b, d, si, d.sI, sk, d.sK, 1);
    dadi_sweep(b, prm, d, d.sK, d.nz, sk, sj, qq_k, cc_k, dual_dt, d.sI, d.nx, d.sJ, d.ny);
    /* T_zeta: back to conservative variables (:1679-1731) and the -1/vol scaling (:1735-1746) */
    const double sqrt2inv = one / sqrt2;
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double uvel = W(c, IVX), vvel = W(c, IVY), wvel = W(c, IVZ);
        double rk1 = half * (sk[c] + sk[c - d.sK]), rk2 = half * (sk[d.N + c] + sk[d.N + c - d.sK]), rk3 = half * (sk[2 * d.N + c] + sk[2 * d.N + c - d.sK]);
        double rk = sqrt(rk1 * rk1 + rk2 * rk2 + rk3 * rk3);
        double uu = uvel * rk1 + vvel * rk2 + wvel * rk3;
        rk1 = rk1 / rk; rk2 = rk2 / rk; rk3 = rk3 / rk;
        double uvw = half * (uvel * uvel + vvel * vvel + wvel * wvel);
        double cijkinv = sqrt(W(c, IRHO) / gam / b->p[c]);
        double alph = W(c, IRHO) * cijkinv * sqrt2inv;
        double xfact = two / cijkinv;
        double ge = gam * W(c, IRHOE) / W(c, IRHO) - (gam - one) * uvw;
        double dw1 = DW(c, 0), dw2 = DW(c, 1), dw3 = DW(c, 2), dw4 = DW(c, 3) * alph, dw5 = DW(c, 4) * alph;
        double a1 = dw1 * rk1 + dw2 * rk2 + dw3 * rk3 + dw4 + dw5;
        double a2 = half * xfact * (dw4 - dw5);
        double a3 = uvw * (rk1 * dw1 + rk2 * dw2 + rk3 * dw3);
        DW(c, 0) = a1;
        DW(c, 1) = a1 * uvel - W(c, IRHO) * (rk3 * dw2 - rk2 * dw3) + a2 * rk1;
        DW(c, 2) = a1 * vvel - W(c, IRHO) * (rk1 * dw3 - rk3 * dw1) + a2 * rk2;
        DW(c, 3) = a1 * wvel - W(c, IRHO) * (rk2 * dw1 - rk1 * dw2) + a2 * rk3;
        DW(c, 4) = a3 + W(c, IRHO) * ((vvel * rk3 - wvel * rk2) * dw1 + (wvel * rk1 - uvel * rk3) * dw2 + (uvel * rk2 - vvel * rk1) * dw3) +
                   (ge + half * xfact * uu / rk) * dw4 + (ge - half * xfact * uu / rk) * dw5;
    }
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double volfact = -one / b->vol[c];
        for (int l = 0; l < 5; l++) DW(c, l) = DW(c, l) * volfact;
    }
}

/* executeDADIStep: src/solver/smoothers.F90:425-693 (steady, fine level) */
void orc_dadi_step(const OrcBlock* b, const AdfbParams* prm0, int nSub, const AdfbSubface* sf) {
    Dims d = dims_of(b);
    /* currentCfl = cflCoarse unless currentLevel == 1 (smoothers.F90:469-472, residuals.F90:1113-1116); second halos
       only on the ground level (smoothers.F90:463-467) */
    AdfbParams prmL = *prm0;
    if (b->level > 1) prmL.cfl = prm0->cflCoarse;
    const AdfbParams* prm = &prmL;
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double dt = -prm->cfl * b->dtl[c] * b->vol[c];
        for (int l = 0; l < 5; l++) DW(c, l) = DW(c, l) * dt;
    }
    orc_compute_dw_dadi(b, prm);
    if (prm->resAveraging == 1) orc_residual_averaging(b, prm); /* rkStage = 0: `alternate` never smooths */
    double gm1 = prm->gammaInf - one;
    for (int k = 2; k <= d.kl; k++) for (int j = 2; j <= d.jl; j++) for (int i = 2; i <= d.il; i++) {
        long c = IDX(i, j, k);
        double ovr = one / W(c, IRHO);
        double v2 = W(c, IVX) * W(c, IVX) + W(c, IVY) * W(c, IVY) + W(c, IVZ) * W(c, IVZ);
        double dp = (ovr * b->p[c] + zero - gm1 * (ovr * W(c, IRHOE) - v2)) * DW(c, IRHO) +
                    gm1 * (DW(c, IRHOE) - W(c, IVX) * DW(c, IMX) - W(c, IVY) * DW(c, IMY) - W(c, IVZ) * DW(c, IMZ));
        double ru = W(c, IRHO) * W(c, IVX) - DW(c, IMX);
        double rv = W(c, IRHO) * W(c, IVY) - DW(c, IMY);
        double rw = W(c, IRHO) * W(c, IVZ) - DW(c, IMZ);
        W(c, IRHO) = W(c, IRHO) - DW(c, IRHO);
        W(c, IRHO) = dmax(W(c, IRHO), 1.e-4 * prm->rhoInf);
        ovr = one / W(c, IRHO);
        W(c, IVX) = ovr * ru; W(c, IVY) = ovr * rv; W(c, IVZ) = ovr * rw;
        b->p[c] = b->p[c] - dp;
        b->p[c] = dmax(b->p[c], 1.e-4 * prm->pInfCorr);
    }
    orc_etot(b, prm, 2, d.il, 2, d.jl, 2, d.kl);
    orc_lam_viscosity(b, prm, 0);
    orc_eddy_viscosity(b, prm, 0);
    orc_apply_flow_bc(b, prm, nSub, sf, b->level > 1 ? 0 : 1);
}

/* ------------------------------------------------------------------------ */
/* wallIntegrationFace, src/solver/surfaceIntegrations.F90:406-881: pressure and viscous force / moment sums of
   the wall subfaces.  BCPointers planes (setBCPointers with spatialPointers): pp2 / pp1 = first interior / first
   halo pressure, ssi = face normal of the wall face, xx = its node coordinates, fact = -1 on min faces.  Face cells are
   weighted by max(BCData%iblank, 0) of the subface (sf->iblank, NULL == 1), not by the volume iblank.
   Owned face cells only (inBeg+1:inEnd): 2..l of the two in-plane directions. */
static double surface_blank(const AdfbSubface* sf, int ia, int jb) {
    if (!sf->iblank) return one;
    return dmax((double)sf->iblank[(ia - sf->icBeg) + (sf->icEnd - sf->icBeg + 1) * (jb - sf->jcBeg)], zero);
}
void orc_wall_forces(const OrcBlock* b, const AdfbParams* prm, int nSub, const AdfbSubface* sfs, const double refPoint[3],
                     double pRef, double out[12]) {
    Dims d = dims_of(b);
    for (int q = 0; q < 12; q++) out[q] = zero;
    for (int n = 0; n < nSub; n++) {
        const AdfbSubface* sf = &sfs[n];
        int viscWall = sf->bcType == ADFB_BC_NSWALL_ADIABATIC || sf->bcType == ADFB_BC_NSWALL_ISOTHERMAL;
        if (!viscWall && sf->bcType != ADFB_BC_EULERWALL) continue;
        Face f = face_of(d, sf->faceId);
        int dir = (sf->faceId - 1) / 2, isMin = (sf->faceId % 2) == 1;
        double fact = isMin ? -one : one;
        const double* s = dir == 0 ? b->si : (dir == 1 ? b->sj : b->sk);
        long sd = dir == 0 ? d.sI : (dir == 1 ? d.sJ : d.sK);
        int la = (f.sa == d.sI) ? d.il : (f.sa == d.sJ ? d.jl : d.kl);
        int lb = (f.sb == d.sJ) ? d.jl : d.kl;
        int a0 = sf->icBeg < 2 ? 2 : sf->icBeg, a1 = sf->icEnd > la ? la : sf->icEnd;
        int b0 = sf->jcBeg < 2 ? 2 : sf->jcBeg, b1 = sf->jcEnd > lb ? lb : sf->jcEnd;
        double Fp[3] = {0, 0, 0}, Fv[3] = {0, 0, 0}, Mp[3] = {0, 0, 0}, Mv[3] = {0, 0, 0};
        for (int jb_ = b0; jb_ <= b1; jb_++) for (int ia = a0; ia <= a1; ia++) {
            long q = ia * f.sa + jb_ * f.sb;
            long c1 = f.off[1] + q, c2 = f.off[2] + q;
            long cf = isMin ? c1 : c2;   /* face index: face between halo and interior cell */
            (void)sd;
            double pm1 = fact * (half * (b->p[c2] + b->p[c1]) - prm->pInf) * pRef;
            /* face centre: the four nodes of the face; node (ia, jb) is the upper one, the lower ones are -sa, -sb */
            double xc[3];
            for (int m = 0; m < 3; m++)
                xc[m] = fourth * (X(cf - f.sa - f.sb, m) + X(cf - f.sb, m) + X(cf - f.sa, m) + X(cf, m));
            double blk = surface_blank(sf, ia, jb_);
            double fx = pm1 * s[cf], fy = pm1 * s[d.N + cf], fz = pm1 * s[2 * d.N + cf];
            double rx = xc[0] - refPoint[0], ry = xc[1] - refPoint[1], rz = xc[2] - refPoint[2];
            Fp[0] += fx * blk; Fp[1] += fy * blk; Fp[2] += fz * blk;
            Mp[0] += (ry * fz - rz * fy) * blk; Mp[1] += (rz * fx - rx * fz) * blk; Mp[2] += (rx * fy - ry * fx) * blk;
        }
        if (viscWall && b->wallTau) {
            const double* t = b->wallTau + (long)dir * 9 * d.N;
            for (int jb_ = b0; jb_ <= b1; jb_++) for (int ia = a0; ia <= a1; ia++) {
                long q = ia * f.sa + jb_ * f.sb;
                long c1 = f.off[1] + q, c2 = f.off[2] + q;
                long cf = isMin ? c1 : c2;
                double blk = surface_blank(sf, ia, jb_);
                double txx = t[cf], tyy = t[d.N + cf], tzz = t[2 * d.N + cf], txy = t[3 * d.N + cf], txz = t[4 * d.N + cf],
                       tyz = t[5 * d.N + cf];
                double s1 = s[cf], s2 = s[d.N + cf], s3 = s[2 * d.N + cf];
                double fx = -fact * (txx * s1 + txy * s2 + txz * s3) * pRef;
                double fy = -fact * (txy * s1 + tyy * s2 + tyz * s3) * pRef;
                double fz = -fact * (txz * s1 + tyz * s2 + tzz * s3) * pRef;
                double xc[3];
                for (int m = 0; m < 3; m++)
                    xc[m] = fourth * (X(cf - f.sa - f.sb, m) + X(cf - f.sb, m) + X(cf - f.sa, m) + X(cf, m));
                double rx = xc[0] - refPoint[0], ry = xc[1] - refPoint[1], rz = xc[2] - refPoint[2];
                Fv[0] += fx * blk; Fv[1] += fy * blk; Fv[2] += fz * blk;
                Mv[0] += (ry * fz - rz * fy) * blk; Mv[1] += (rz * fx - rx * fz) * blk; Mv[2] += (rx * fy - ry * fx) * blk;
            }
        }
        for (int m = 0; m < 3; m++) { out[m] += Fp[m]; out[3 + m] += Fv[m]; out[6 + m] += Mp[m]; out[9 + m] += Mv[m]; }
    }
}

/* orphanAverage (src/utils/haloExchange.F90:201-354): every overset orphan takes the average of its (up to six)
 * face neighbours with iblank == 1; with no such neighbour it falls back to the free stream (wInf, pInfCorr, muInf,
 * eddyVisInfRatio * muInf).  orphans = (3, nOrphans) cell indices (i, j, k); variables w(wStart:wEnd) [1-based],
 * p / rlv / rev when asked (gamma is constant here). */
void orc_orphan_average(const OrcBlock* b, const AdfbParams* prm, int nOrphans, const int32_t* orphans, int wStart, int wEnd,
                        int calcPressure, int calcLamVis, int calcEddyVis, double muInf, double eddyVisInfRatio) {
    const int ib = b->nx + 3, jb = b->ny + 3, kb = b->nz + 3;
    const long NI = ib + 1, NJ = jb + 1, N = NI * NJ * (kb + 1);
    double* w = (double*)b->w; double* p = (double*)b->p; double* rlv = (double*)b->rlv; double* rev = (double*)b->rev;
    const int32_t* iblank = (const int32_t*)b->iblank;
    for (int n = 0; n < nOrphans; n++) {
        const int oi = orphans[3 * n], oj = orphans[3 * n + 1], ok = orphans[3 * n + 2];
        const long c = oi + NI * (oj + NJ * (long)ok);
        int nAvg = 0;
        for (int l = wStart; l <= wEnd; l++) w[(l - 1) * N + c] = 0.0;
        if (calcPressure) p[c] = 0.0;
        if (calcLamVis) rlv[c] = 0.0;
        if (calcEddyVis) rev[c] = 0.0;
        for (int m = 0; m < 3; m++)
            for (int i = -1; i <= 1; i += 2) {
                const int ni = oi + (m == 0 ? i : 0), nj = oj + (m == 1 ? i : 0), nk = ok + (m == 2 ? i : 0);
                if (ni < 0 || ni > ib || nj < 0 || nj > jb || nk < 0 || nk > kb) continue;
                const long cn = ni + NI * (nj + NJ * (long)nk);
                if (iblank[cn] == 1) {
                    nAvg++;
                    for (int l = wStart; l <= wEnd; l++) w[(l - 1) * N + c] = w[(l - 1) * N + c] + w[(l - 1) * N + cn];
                    if (calcPressure) p[c] = p[c] + p[cn];
                    if (calcLamVis) rlv[c] = rlv[c] + rlv[cn];
                    if (calcEddyVis) rev[c] = rev[c] + rev[cn];
                }
            }
        if (nAvg > 0) {
            const double r = (double)nAvg;
            for (int l = wStart; l <= wEnd; l++) w[(l - 1) * N + c] = w[(l - 1) * N + c] / r;
            if (calcPressure) p[c] = p[c] / r;
            if (calcLamVis) rlv[c] = rlv[c] / r;
            if (calcEddyVis) rev[c] = rev[c] / r;
        } else {
            for (int l = wStart; l <= wEnd; l++) w[(l - 1) * N + c] = prm->wInf[l - 1];
            if (calcPressure) p[c] = prm->pInfCorr;
            if (calcLamVis) rlv[c] = muInf;
            if (calcEddyVis) rev[c] = eddyVisInfRatio * muInf;
        }
    }
}
