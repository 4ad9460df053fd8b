/* ref_env.h -- TEST INFRASTRUCTURE ONLY.
 *
 * Environment for oracle/_ref/blockette_ref.c, the C translation (oracle/f90toc.py) of the
 * reference's src/NKSolver/blockette.F90.  The translated routines reference module variables
 * of OTHER reference modules (inputPhysics, inputDiscretization, flowVarRefState, iteration,
 * paramTurb, sa, blockPointers ...).  Those modules are not translated; this header declares
 * the variables as C globals (lower-cased Fortran names; blockPointers names carry the prefix
 * bp_) and ref_env.c defines them and fills them from the test harness.
 *
 * `parameter` constants of src/modules/constants.F90 are NOT restated here: they are generated
 * from the reference file into oracle/_ref/ref_constants.h.
 */
#ifndef ADFB_REF_ENV_H
#define ADFB_REF_ENV_H
#include <stddef.h>
#include "ref_constants.h"

/* flowVarRefState */
extern int nw, nwf, nt1, nt2, viscous, kpresent, eddymodel;
extern double pinfcorr, rhoinf, gammainf, timeref, rgas, tref;
/* inputPhysics */
extern int equations, equationmode, turbmodel, turbprod, useqcr, useft2sa, userotationsa;
extern double prandtl, prandtlturb;
/* inputDiscretization */
extern int spacediscr, orderturb, limiter, precond, riemann, riemanncoarse, approxsa;
extern double vis2coarse;
extern double vis2, vis4, sigma, adis, acousticscalefactor, kappacoef;
/* inputIteration */
extern int usedisscontinuation;
extern double disscontmagnitude, disscontmidpoint, disscontsharpness;
extern double turbresscale[4];
/* iteration */
extern int currentlevel, groundlevel;
extern double rfil, totalr0, totalr;
/* more of inputPhysics / inputIteration / inputUnsteady / iteration / block used by the smoothers */
extern int cpmodel, rkstage, resaveraging, bp_ndom, exchangepressureearly, lowspeedpreconditioner;
extern double gammaconstant, musuthdim, tsuthdim, ssuthdim, muref, pinf;
extern double cfl, cflcoarse, cfllimit, smoop, deltat;
extern double etark[6], cdisrk[6], coeftime[8];
extern double *bp_wn, *bp_pn, *bp_scratch;
extern double *bp_bmti1, *bp_bmti2, *bp_bmtj1, *bp_bmtj2, *bp_bmtk1, *bp_bmtk2;
extern int turbrelax;
extern double alfaturb;
/* inputTimeSpectral, oversetData, turbMod */
extern int ntimeintervalsspectral, oversetpresent, secondord;
/* paramTurb (SA constants) */
extern double rsak, rsacb1, rsacb2, rsacb3, rsacv1, rsacw1, rsacw2, rsacw3, rsact1, rsact2, rsact3, rsact4, rsacrot;
/* blockPointers: extents and arrays of the current block, uniform box (0:ib,0:jb,0:kb) */
extern int bp_nx, bp_ny, bp_nz, bp_il, bp_jl, bp_kl, bp_ie, bp_je, bp_ke, bp_ib, bp_jb, bp_kb;
extern int bp_addgridvelocities, bp_righthanded, bp_sectionid, bp_blockismoving, bp_nbkglobal;
extern double *bp_w, *bp_p, *bp_gamma, *bp_rlv, *bp_rev, *bp_vol, *bp_volref, *bp_d2wall, *bp_shocksensor;
extern double *bp_x, *bp_si, *bp_sj, *bp_sk, *bp_sfacei, *bp_sfacej, *bp_sfacek;
extern double *bp_dw, *bp_fw, *bp_dtl, *bp_aa, *bp_radi, *bp_radj, *bp_radk;
extern double *bp_ux, *bp_uy, *bp_uz, *bp_vx, *bp_vy, *bp_vz, *bp_wx, *bp_wy, *bp_wz, *bp_qx, *bp_qy, *bp_qz;
extern int *bp_iblank, *bp_pori, *bp_porj, *bp_pork;
/* overset orphans of the block (blockPointers nOrphans, orphans(3, nOrphans)) and the free-stream viscosities orphanAverage falls back to */
extern int bp_norphans, *bp_orphans;
extern double muinf, eddyvisinfratio;
extern double *bp_rotmatrixi, *bp_rotmatrixj, *bp_rotmatrixk;

/* utils procedures the translated code calls */
int getcorrectfork(void);                           /* src/utils/utils.F90 getCorrectForK */
void terminate(const char* routine, const char* msg); /* src/utils/utils.F90 terminate */

/* boundary-condition bookkeeping of the current block (blockPointers nBocos, BCType, BCFaceID, BCData) */
extern int bp_nbocos, bp_nviscbocos, bp_bctype[64], bp_bcfaceid[64];
extern int viscwallbctreatment, eulerwallbctreatment, outflowtreatment, wallfunctions, hscalinginlet;
extern double winf[10];
extern int lumpeddiss, viscpc, spacediscrcoarse, smoother, nrkstages, nsubiterations, subit, radiineededfine, radiineededcoarse, dirscaling;   /* iteration / inputDiscretization / inputIteration */
extern double* bp_wr;
extern double monloc[16];   /* module monitor: local residual sums */
extern double *bp_s;
extern int *bp_globalcell;
extern double *bp_bvti1, *bp_bvti2, *bp_bvtj1, *bp_bvtj2, *bp_bvtk1, *bp_bvtk2;
/* BCData(nn): cell range of the subface and its per-face data, Fortran order (icBeg:icEnd, jcBeg:jcEnd[, 3]) */
typedef struct {
    int icbeg, icend, jcbeg, jcend;
    double *norm, *rface, *uslip, *tns_wall;
    int inbeg, inend, jnbeg, jnend; /* node range of the subface (owned face cells are inBeg+1:inEnd) */
    int* iblank;                    /* BCData%iblank: surface blanking of the face cells, (icBeg:icEnd, jcBeg:jcEnd) */
    double* tau;                    /* viscSubface%tau(:,:,6), same layout */
    /* in/outflow data */
    double *ps, *rho, *velx, *vely, *velz, *ptinlet, *ttinlet, *htinlet, *flowxdirinlet, *flowydirinlet, *flowzdirinlet, *turbinlet;
    int subsonicinlettreatment, pad_;
} RefSubface;
extern RefSubface bcd[64];
static inline int bcd_icbeg(int nn) { return bcd[nn - 1].icbeg; }
static inline int bcd_icend(int nn) { return bcd[nn - 1].icend; }
static inline int bcd_jcbeg(int nn) { return bcd[nn - 1].jcbeg; }
static inline int bcd_jcend(int nn) { return bcd[nn - 1].jcend; }
static inline long bcd_off(int nn, int i, int j) {
    const RefSubface* s = &bcd[nn - 1];
    return (i - s->icbeg) + (long)(s->icend - s->icbeg + 1) * (j - s->jcbeg);
}
static inline long bcd_size(int nn) {
    const RefSubface* s = &bcd[nn - 1];
    return (long)(s->icend - s->icbeg + 1) * (s->jcend - s->jcbeg + 1);
}
static inline double bcd_norm(int nn, int i, int j, int l) { return bcd[nn - 1].norm[bcd_off(nn, i, j) + (l - 1) * bcd_size(nn)]; }
static inline double bcd_uslip(int nn, int i, int j, int l) { return bcd[nn - 1].uslip[bcd_off(nn, i, j) + (l - 1) * bcd_size(nn)]; }
static inline double bcd_rface(int nn, int i, int j) { return bcd[nn - 1].rface[bcd_off(nn, i, j)]; }
#define BCD_SCALAR(name) static inline double bcd_##name(int nn, int i, int j) { return bcd[nn - 1].name[bcd_off(nn, i, j)]; }
BCD_SCALAR(ps) BCD_SCALAR(rho) BCD_SCALAR(velx) BCD_SCALAR(vely) BCD_SCALAR(velz) BCD_SCALAR(ptinlet) BCD_SCALAR(ttinlet)
BCD_SCALAR(htinlet) BCD_SCALAR(flowxdirinlet) BCD_SCALAR(flowydirinlet) BCD_SCALAR(flowzdirinlet)
static inline int bcd_subsonicinlettreatment(int nn) { return bcd[nn - 1].subsonicinlettreatment; }
/* BCData%turbInlet(i, j, nt1:nt2): one turbulence variable (SA) */
static inline double bcd_turbinlet(int nn, int i, int j, int l) { (void)l; return bcd[nn - 1].turbinlet[bcd_off(nn, i, j)]; }
static inline int bcd_inbeg(int nn) { return bcd[nn - 1].inbeg; }
static inline int bcd_inend(int nn) { return bcd[nn - 1].inend; }
static inline int bcd_jnbeg(int nn) { return bcd[nn - 1].jnbeg; }
static inline int bcd_jnend(int nn) { return bcd[nn - 1].jnend; }
static inline int bcd_iblank(int nn, int i, int j) { return bcd[nn - 1].iblank[bcd_off(nn, i, j)]; }
static inline double bcd_cptarget(int nn, int i, int j) { (void)nn; (void)i; (void)j; return 0.0; } /* Cp-target cost function: unused */
static inline double vsf_tau(int nn, int i, int j, int l) { return bcd[nn - 1].tau[bcd_off(nn, i, j) + (l - 1) * bcd_size(nn)]; }
static inline double bcd_tns_wall(int nn, int i, int j) { return bcd[nn - 1].tns_wall[bcd_off(nn, i, j)]; }

/* inputPhysics / inputCostFunctions / flowVarRefState data read by wallIntegrationFace */
extern int spectralsol, computesepsensorks, computecavitation, cavexponent, rvfn;
extern double pref, lref, machcoef, cpmin_rho, cavitationnumber, cavsensorsharpness, cavsensoroffset;
extern double sepsensorsharpness, sepsensoroffset, sepsensorkssharpness, sepsensorksphi, sepsensorksoffset, sepsenmaxrho;
extern double veldirfreestream[3], pointref[3], momentaxis[6], cpmin_family[4], sepsenmaxfamily[4];

/* multigrid (src/solver/multiGrid.F90): w1/p1 and the restriction / interpolation tables of the current block, the
   OTHER level's block that transferToCoarseGrid (fine: fl_) and transferToFineGrid (coarse: cl_) reach through
   flowDoms(nn, level, sps), and the coarse block's BCData (cbcd) */
extern double *bp_w1, *bp_p1, *bp_mgiweight, *bp_mgjweight, *bp_mgkweight;
extern int *bp_mgifine, *bp_mgjfine, *bp_mgkfine, *bp_mgicoarse, *bp_mgjcoarse, *bp_mgkcoarse;
extern int sh_ib, sh_jb, sh_kb; /* box of the (finest-level) arrays that dw, fw, dtl, rad*, rlv, gamma, wn, pn, scratch point at */
extern int fl_ib, fl_jb, fl_kb, cl_il, cl_jl, cl_kl, cl_ie, cl_je, cl_ke, cl_ib, cl_jb, cl_kb, cl_nbocos, mgboundcorr;
extern double *fl_w, *fl_p, *fl_vol, *fl_rev, *fl_w1, *fl_p1, *cl_w, *cl_p, *cl_vol, *cl_rev, *cl_w1, *cl_p1;
extern int *fl_iblank, *cl_iblank, cl_bctype[64], cl_bcfaceid[64];
extern double fcoll;
extern RefSubface cbcd[64];
static inline int cbcd_icbeg(int nn) { return cbcd[nn - 1].icbeg; }
static inline int cbcd_icend(int nn) { return cbcd[nn - 1].icend; }
static inline int cbcd_jcbeg(int nn) { return cbcd[nn - 1].jcbeg; }
static inline int cbcd_jcend(int nn) { return cbcd[nn - 1].jcend; }
static inline double cbcd_norm(int nn, int i, int j, int l) {
    const RefSubface* s = &cbcd[nn - 1];
    const long na = s->icend - s->icbeg + 1, nb = s->jcend - s->jcbeg + 1;
    return s->norm[(i - s->icbeg) + na * (j - s->jcbeg) + (l - 1) * na * nb];
}
/* setPointers(nn, level, sps): the harness registers a callback that rebinds bp_* and bcd to the block of `level` */
extern void (*setpointers_hook)(int level);
void solverutils_timestep(int* onlyradii);
void turbbcroutines_applyallturbbc(int* secondhalo);

/* ANK (module ANKSolver of src/NKSolver/NKSolvers.F90): option code of ANK_charTimeStepType ('None' 0, 'VLR' 1,
   'Turkel' 2), free-stream Mach number, the PETSc vectors wVec / deltaW as arrays, nState x nState helpers */
extern int ank_chartimestepcode, ank_nvec;
extern double ank_machinf, *ank_wvec, *ank_dvec;
void ank_matmul(double* a, double* b, double* c);     /* c = MATMUL(a, b) */
void ank_matmul_nt(double* a, double* b, double* c);  /* c = MATMUL(a, TRANSPOSE(b)) */

/* executeMGCycle (src/solver/multiGrid.F90:825-955): iteration%cycling / nStepsCycling, the turbulence solve of
   src/turbulence/turbAPI.F90:4-95 (SA: nSubIterTurb x sa_block) and computeUtau (wall functions: off) */
extern int nstepscycling, cycling[256], approxtotalits, nsubiterturb;
void solverutils_computeutau(void);
void turbsolveddadi(void);

/* driver-level procedures outside the translated set (no-op stubs, see ref_env.c) */
void setpointers(int* nn, int* level, int* sps);
void whalo1(int* level, int* start, int* end, int* commpressure, int* commgamma, int* commviscous);
void whalo2(int* level, int* start, int* end, int* commpressure, int* commgamma, int* commviscous);

#endif
