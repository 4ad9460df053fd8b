/*
 * adflow_b200.h -- C ABI of libadflow_b200.so
 *
 * H100-native (sm_90a) implementation of the per-block residual / smoother /
 * matrix-free Jacobian-vector hot path of mdolab/adflow.  The reference has no
 * FFI seam around this path (SURVEY.md section 8b): its L2 routines are
 * argument-less Fortran module procedures acting on module-global block
 * pointers.  Each entry point below names the reference routine (file:line,
 * relative to the reference tree) whose body it replaces; INTEGRATION.md shows
 * the ISO_C_BINDING interface block a maintainer adds on the Fortran side.
 *
 * Conventions
 *  - every function returns 0 on success, non-zero on failure; the message is
 *    available from adfb_last_error().  The Fortran caller maps non-zero to
 *    `call terminate(routine, msg)` (src/utils/utils.F90:501).
 *  - all reals are IEEE double (src/modules/precision.F90:74-81 realType),
 *    ints are 32 bit (intType), porosities are int8 (porType).
 *  - host arrays are Fortran column-major with the reference's own extents and
 *    lower bounds; they are only read/written during the call (no retained
 *    pointers).  Extents for a block of nx*ny*nz owned cells
 *    (il=nx+1, ie=nx+2, ib=nx+3; idem j,k; src/modules/block.F90:209-223):
 *       w(0:ib,0:jb,0:kb,1:nw) p,rlv,rev,vol,volRef,dw(0:ib,0:jb,0:kb[,1:nw])
 *       iblank(0:ib,0:jb,0:kb) int32
 *       x(0:ie,0:je,0:ke,3)
 *       sI(0:ie,1:je,1:ke,3) sJ(1:ie,0:je,1:ke,3) sK(1:ie,1:je,0:ke,3)
 *       porI(1:il,2:jl,2:kl) porJ(2:il,1:jl,2:kl) porK(2:il,2:jl,1:kl) int8
 *       d2Wall(2:il,2:jl,2:kl)
 *       dtl,radI,radJ,radK(1:ie,1:je,1:ke)
 *  - not re-entrant; called from the rank's only thread (the reference is
 *    single threaded per MPI rank).  One process <-> one GPU.
 *  - the library has NO CPU fallback: every entry point fails with an error if
 *    no CUDA device is usable.
 */
#ifndef ADFLOW_B200_H
#define ADFLOW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* variable slots, src/modules/constants.F90:34-40 (1-based in Fortran) */
enum { ADFB_IRHO = 0, ADFB_IVX = 1, ADFB_IVY = 2, ADFB_IVZ = 3, ADFB_IRHOE = 4, ADFB_ITU1 = 5 };

/* equations, src/modules/constants.F90 (EulerEquations/NSEquations/RANSEquations) */
enum { ADFB_EULER = 1, ADFB_NS = 2, ADFB_RANS = 3 };
/* spaceDiscr */
enum { ADFB_DISS_SCALAR = 1, ADFB_DISS_MATRIX = 2, ADFB_UPWIND = 4 };
/* turbProd */
enum { ADFB_PROD_STRAIN = 1, ADFB_PROD_VORTICITY = 2 };
/* limiter for the upwind scheme (inputDiscretization%limiter) */
enum { ADFB_LIM_FIRSTORDER = 0, ADFB_LIM_NONE = 1, ADFB_LIM_VANALBADA = 2, ADFB_LIM_MINMOD = 3 };
/* porosity codes, src/modules/constants.F90:28-30 */
enum { ADFB_NOFLUX = -1, ADFB_BOUNDFLUX = 0, ADFB_NORMALFLUX = 1 };
/* BC types handled on device (subset of src/modules/constants.F90:257-282) */
enum {
    ADFB_BC_SYMM = 1,
    ADFB_BC_NSWALL_ADIABATIC = 2,
    ADFB_BC_FARFIELD = 3,
    ADFB_BC_EULERWALL = 4,
    ADFB_BC_EXTRAP = 5,
    ADFB_BC_NSWALL_ISOTHERMAL = 6,
    ADFB_BC_SUBSONIC_OUTFLOW = 7,   /* bcSubsonicOutflow (also MassBleedOutflow), needs ps */
    ADFB_BC_SUBSONIC_INFLOW = 8,    /* bcSubsonicInflow: totalConditions (ptInlet, ttInlet, htInlet, flow?dirInlet) or massFlow (rho, vel?) */
    ADFB_BC_SUPERSONIC_INFLOW = 9,  /* bcSupersonicInflow: rho, velx, vely, velz, ps prescribed */
    ADFB_BC_SUPERSONIC_OUTFLOW = 10, /* bcExtrap with outflowTreatment (constant or linear extrapolation) */
    ADFB_BC_SYMMPOLAR = 11          /* bcSymmPolar1stHalo/2ndHalo (BCRoutines.F90:332-486): singular (polar) line, the
                                       mirror direction is the diagonal of the collapsed face, taken from the mesh x */
};
/* block faces, reference order iMin..kMax (src/modules/constants.F90 iMin=1..kMax=6) */
enum { ADFB_IMIN = 1, ADFB_IMAX = 2, ADFB_JMIN = 3, ADFB_JMAX = 4, ADFB_KMIN = 5, ADFB_KMAX = 6 };

/* residual flags == blocketteRes optional logicals, src/NKSolver/blockette.F90:70-164 */
enum {
    ADFB_RES_DISS_APPROX = 1,     /* useDissApprox   */
    ADFB_RES_VISC_APPROX = 2,     /* useViscApprox   */
    ADFB_RES_UPDATE_INTERMED = 4, /* useUpdateIntermed: also store dtl, radI/J/K */
    ADFB_RES_FLOW = 8,            /* useFlowRes      */
    ADFB_RES_TURB = 16,           /* useTurbRes      */
    ADFB_RES_STORE_WALL = 32,     /* useStoreWall    */
    ADFB_RES_SKIP_PREAMBLE = 64   /* core only: skip p/rlv/rev + BCs + halo exchange
                                     (== calling blocketteResCore directly) */
};

/*
 * All scalar module globals the hot path reads, passed by value
 * (replaces inputDiscretization, inputPhysics, flowVarRefState, paramTurb,
 * inputIteration module state; SURVEY.md section 5 "Config / flags").
 */
typedef struct AdfbParams {
    /* reference state, src/initFlow/initializeFlow.F90:10-182 (referenceState) */
    double gammaInf;   /* == gammaConstant (cpConstant model only) */
    double RGas;
    double pInfCorr;
    double rhoInf;
    double wInf[6];    /* rho, u, v, w, rhoE, nuTilde of the free stream */
    double pInf;
    /* Sutherland, non-dimensional: muSuthDim/muRef, TSuthDim/Tref, SSuthDim/Tref
       (src/utils/flowUtils.F90:1241-1243) */
    double muSuth, TSuth, SSuth;
    double prandtl, prandtlTurb;
    /* JST, src/inputParam/inputParamRoutines.F90:3823-3833 + pyADflow defaults */
    double vis2, vis4, adis, acousticScaleFactor;
    double kappaCoef;  /* MUSCL kappa for the upwind scheme */
    /* SA model, src/modules/paramTurb.F90:8-20 */
    double rsaK, rsaCb1, rsaCb2, rsaCb3, rsaCv1, rsaCw1, rsaCw2, rsaCw3, rsaCt3, rsaCt4, rsaCrot;
    /* smoothers, src/inputParam/inputParamRoutines.F90:3576-3633 */
    double cfl, cflCoarse;
    double etaRK[6], cdisRK[6];
    double alfaTurb;      /* DD-ADI under-relaxation, inputParamRoutines.F90:3908 */
    double turbResScale;  /* NKSolvers.F90:1295-1307 */
    double cflLimit, smoop; /* residual averaging, residuals.F90:1850-1893 */
    double sigma;           /* dissipationLumpingParameter of the *Approx dissipation (blockette.F90:4416) */
    /* multigrid: inputDiscretization vis2Coarse (first-order coarse-level dissipation, fluxes.F90:4977-5203) and
       inputIteration fcoll (relaxation of the restricted residual, multiGrid.F90:306-317) */
    double vis2Coarse, fcoll;
    /* integer switches */
    int32_t equations;    /* ADFB_EULER / NS / RANS */
    int32_t spaceDiscr;   /* ADFB_DISS_SCALAR ... */
    int32_t nRKStages;
    int32_t turbProd;
    int32_t useQCR;
    int32_t useft2SA;
    int32_t useRotationSA;
    int32_t approxSA;
    int32_t secondOrdTurb; /* turbMod%secondOrd, turbUtils.F90:828 ff. */
    int32_t limiter;
    int32_t resAveraging;  /* 0 never, 1 always, 2 alternate */
    int32_t nSubiterTurb;
    int32_t wallBCConstantPressure; /* viscWallBCTreatment == constantPressure */
    int32_t reserved;
    int32_t hScalingInlet;         /* inputDiscretization hScalingInlet (subsonic inflow, total conditions) */
    int32_t outflowLinearExtrapol; /* outflowTreatment == linExtrapol (default constantExtrapol), supersonic outflow */
    int32_t mgBoundCorr;           /* 0 = bcDirichlet0 (default), 1 = bcNeumann0: boundary halos of the interpolated corrections */
    int32_t spaceDiscrCoarse;      /* coarse-level discretisation: ADFB_DISS_SCALAR or ADFB_DISS_MATRIX on levels > 1 */
} AdfbParams;

/* One boundary subface of a block, mirroring BCDataType (src/modules/block.F90:52-156)
   for the BC classes handled on device.  Ranges are the *cell* ranges icBeg:icEnd,
   jcBeg:jcEnd of BCData(nn) in the two in-plane directions (utils.F90:895-900). */
typedef struct AdfbSubface {
    int32_t bcType;   /* ADFB_BC_* */
    int32_t faceId;   /* ADFB_IMIN .. ADFB_KMAX */
    int32_t icBeg, icEnd, jcBeg, jcEnd;
    /* optional per-face arrays, NULL for defaults; extents (icBeg:icEnd, jcBeg:jcEnd[,3]) */
    const double* norm;   /* unit outward normal BCData%norm, required for symm / wall / farfield */
    const double* rface;  /* BCData%rface (grid normal velocity), NULL == 0 */
    const double* uSlip;  /* BCData%uSlip(:,:,3), NULL == 0 */
    const double* TNSWall; /* isothermal walls only */
    /* in/outflow data of BCData (src/modules/block.F90:100-140), extents (icBeg:icEnd, jcBeg:jcEnd); NULL if unused */
    const double* ps;                       /* static pressure: subsonic outflow, supersonic inflow */
    const double *rho, *velx, *vely, *velz; /* supersonic inflow, subsonic inflow with massFlow treatment */
    const double *ptInlet, *ttInlet, *htInlet, *flowXdirInlet, *flowYdirInlet, *flowZdirInlet; /* total conditions */
    const double* turbInlet;                /* BCData%turbInlet(:,:,nt1:nt2): turbulence variable at inflow faces */
    int32_t subsonicInletTreatment;         /* 1 totalConditions, 2 massFlow (constants.F90:237-238) */
    int32_t pad_;
} AdfbSubface;

/* ---- life cycle ---------------------------------------------------------- */
/* one MPI rank <-> one GPU <-> one NCCL rank.  ncclUniqueId may be NULL when
   nranks == 1.  Replaces nothing in the reference (no device exists there);
   called after partitionAndReadGrid (adflow/pyADflow.py:236). */
int adfb_init(int device, const void* ncclUniqueId, int rank, int nranks);
/* releases every device resource; the counterpart of releaseMemoryPart1/2 (src/utils/utils.F90) at the end of a run */
int adfb_finalize(void);
/* rank 0 calls this and broadcasts the 128 bytes over its own transport (MPI_Bcast
   in the Fortran host, torch.distributed in the Python harness). */
int adfb_get_unique_id(void* out128);
/* message of the last failing call on this rank; the Fortran side hands it to terminate() (src/utils/utils.F90:501) */
int adfb_last_error(char* buf, int n);
/* number of visible CUDA devices (used to map local MPI ranks to GPUs; no counterpart in the reference) */
int adfb_device_count(void);

/* ---- data model (src/modules/block.F90:205-752 blockType) ----------------- */
/* after allocMemFlovarPart2 (src/initFlow/initializeFlow.F90:686-722) */
int adfb_block_create(int blk, int level, int nx, int ny, int nz, int nw, int rightHanded);
/* deallocation of one flowDoms(nn, level, sps) entry (deallocateBlock, src/utils/utils.F90) */
int adfb_block_destroy(int blk);
/* after preprocessing / each mesh warp (updateGeometryInfo).  si/sj/sk may be NULL:
   they are then computed on the device from x with the blockette `metrics`
   formula (src/NKSolver/blockette.F90:854-960).  d2Wall may be NULL for Euler/NS. */
int adfb_block_set_geometry(int blk, const double* x, const double* si, const double* sj,
                            const double* sk, const double* vol, const double* volRef,
                            const double* d2Wall, const int8_t* porI, const int8_t* porJ,
                            const int8_t* porK, const int32_t* iblank);
/* after updateBCDataAllLevels (src/bcdata/BCData.F90): BCData(mm)%norm, rface, uSlip, TNS_Wall, ps, ptInlet ... of block.F90:52-156 */
int adfb_block_set_bc(int blk, int nSub, const AdfbSubface* subfaces);
/* whenever options / AeroProblem change (setOption, _setAeroProblemData in adflow/pyADflow.py; the module variables of
   src/modules/inputParam.F90, flowVarRefState, paramTurb that referenceState, src/initFlow/initializeFlow.F90:10-182, fills) */
int adfb_set_params(const AdfbParams* prm);

/* ---- explicit sync points (NKSolvers.F90:1378-1485 getStates/setStates/getRes) */
int adfb_upload_state(int blk, const double* w, const double* p);
int adfb_download_state(int blk, double* w, double* p, double* rlv, double* rev);
int adfb_upload_visc(int blk, const double* rlv, const double* rev);
int adfb_download_residual(int blk, double* dw);
int adfb_download_intermed(int blk, double* dtl, double* radI, double* radJ, double* radK);

/* Vector forms used by the Python layer and PETSc (NKSolvers.F90:1378-1485):
   ordering = for block, for k, for j, for i, for l=1..nw (AoS per owned cell).
   adfb_get_states <- getStates, adfb_set_states <- setStates (no clipping),
   adfb_get_res <- the gather loop of getRes (dw/volRef, :1432-1448; it does not
   evaluate the residual: call adfb_residual first). n = total vector length. */
int adfb_get_states(double* states, long long n);
int adfb_set_states(const double* states, long long n);
int adfb_get_res(double* res, long long n);
long long adfb_state_size(void);

/* ---- the hot path --------------------------------------------------------- */
/* replaces blocketteRes body, src/NKSolver/blockette.F90:199-283 */
int adfb_residual(int level, unsigned flags);
/* Sum of (dw(irho)/vol)^2 and of all (dw/vol)^2 over owned cells of all local
   blocks, all-reduced (getCurrentResidual, NKSolvers.F90:335-370). out[0]=rho, out[1]=total */
int adfb_norms(double out[2]);
/* blocks until the library stream is idle (the reference is synchronous: needed only before timing or host reads
   that bypass the download calls) */
int adfb_synchronize(void);
/* wallIntegrationFace / getForces (src/solver/surfaceIntegrations.F90:406-881, src/warping/getForces.F90):
   out = Fp(3), Fv(3), Mp(3), Mv(3) summed over the wall subfaces (viscous walls: pressure + viscous, Euler walls:
   pressure) of all blocks of `level` on all ranks; moments about refPoint; forces scaled by pRef like the
   reference.  The viscous part needs a preceding adfb_residual(level, flags | ADFB_RES_STORE_WALL). */
int adfb_forces(int level, const double refPoint[3], double pRef, double out[12]);

/* referenceShockSensor (src/adjoint/adjointUtils.F90:1900-1950): freeze the shock sensor
   field (p for Euler, p/rho**gamma otherwise) used by the ADFB_RES_DISS_APPROX variants */
int adfb_reference_shock_sensor(int level);

/* ---- NK matrix-free residual-Jacobian product ------------------------------ */
/* FormFunction_mf (src/NKSolver/NKSolvers.F90:437-461): setW(wVec) with the turbulence
   clip max(1e-6*wInf, .) (:1331-1376), full residual (blocketteRes), setRVec
   (dw/volRef, turbulence rows * turbResScale, :1262-1329).  Host vectors, AoS ordering. */
int adfb_form_function(const double* wVec, double* rVec, long long n);
/* MatMFFDSetBase (NKSolvers.F90:630): keep U and F(U) on the device */
int adfb_mffd_set_base(const double* U, long long n);
/* MatMult of the MFFD shell that replaces MatCreateMFFD (NKSolvers.F90:167):
   y = (F(U + h a) - F(U)) / h, perturbation, residual and difference all on the device.
   h > 0 is used as given; h <= 0 selects PETSc's default Walker-Pernice
   h = sqrt(eps) * sqrt(1 + ||U||) / ||a|| (norms reduced on the device, all-reduced). */
int adfb_mffd_apply(const double* a, double* y, long long n, double h);
/* the same product for vectors that already live on this device (e.g. PETSc VECCUDA arrays from
   VecCUDAGetArrayRead / VecCUDAGetArrayWrite inside the MatShell's MATOP_MULT): no host copies */
int adfb_mffd_apply_device(const double* aDev, double* yDev, long long n, double h);
double adfb_mffd_last_h(void);

/* ---- halo exchange (src/utils/haloExchange.F90) ---------------------------- */
/* Device copy of the 1-to-1 communication pattern commPatternCell_2nd /
   internalCell_2nd (src/modules/communication.F90:85-168, built by
   src/preprocessing/pointMatchedCommPattern.F90).  Lists are (block, i, j, k) int32
   quadruples with the reference's cell indices (0:ib ...), concatenated over the
   neighbour ranks in the order of nbrRank; the send list of rank A towards B must
   enumerate cells in the same order as B's receive list from A (as the reference's
   sendList/recvList do).  donorList/haloList are the same-rank copies
   (internal%donorBlock/donorIndices -> haloBlock/haloIndices). */
int adfb_comm_set_pattern(int level, int nNbr, const int* nbrRank, const int* sendCount, const int* recvCount,
                          const int* sendList, const int* recvList, int nInternal, const int* donorList,
                          const int* haloList);
/* Device copy of the overset communication pattern commPatternOverset / internalOverset
   (src/modules/communication.F90, built by the overset connectivity search).  Same list conventions as
   adfb_comm_set_pattern; a donor entry (block, i, j, k) names the LOW corner of the 2x2x2 donor stencil and
   sendInterp / donorInterp hold its 8 weights per entry in the reference's order (sendList%interp(j,1:8),
   i fastest: (i,j,k), (i+1,j,k), (i,j+1,k), ...), wOversetGeneric src/utils/haloExchange.F90:1471-1654.
   Once set, adfb_halo_exchange (and every call that exchanges halos) runs the overset exchange right after the
   1-to-1 exchange like whalo2 does, followed by orphanAverage on the blocks that carry an orphan list
   (adfb_block_set_orphans). */
int adfb_comm_set_overset(int level, int nNbr, const int* nbrRank, const int* sendCount, const int* recvCount,
                          const int* sendList, const double* sendInterp, const int* recvList, int nInternal,
                          const int* donorList, const double* donorInterp, const int* haloList);
/* Overset orphans of a block (blockPointers nOrphans / orphans(3, nOrphans), set by the overset connectivity,
   src/overset/oversetUtilities.F90:1638-1667): cell indices (i, j, k) with the reference's bounds, 3 * nOrphans ints.
   Every exchange then ends with orphanAverage (src/utils/haloExchange.F90:201-354, called by whalo1 / whalo2 after
   wOverset): an orphan takes the average of its face neighbours with iblank == 1, or the free stream (wInf, pInfCorr,
   muInf, eddyVisInfRatio * muInf: flowVarRefState) when it has none.  nOrphans = 0 removes the list. */
int adfb_block_set_orphans(int blk, int nOrphans, const int32_t* orphans, double muInf, double eddyVisInfRatio);
/* whalo2(level, start, end, commPressure, commGamma, commViscous)
   (src/utils/haloExchange.F90:109-199): w(start:end) [1-based], p, rlv, rev of all
   listed halo cells; grouped ncclSend/ncclRecv over NVLink; then computeEtotBlock on
   the owned cells when both p and rhoE were exchanged (:174-197). */
int adfb_halo_exchange(int level, int start, int end, int commPressure, int commGamma, int commViscous);

/* ---- smoothers ------------------------------------------------------------- */
/* applyAllBC(secondHalo) (src/solver/BCRoutines.F90:57-222); withTurb != 0 first runs
   bcTurbTreatment + applyAllTurbBCThisBlock (src/turbulence/turbBCRoutines.F90:49,662) */
int adfb_apply_bcs(int level, int secondHalo, int withTurb);
/* timeStep(onlyRadii): spectral radii radI/J/K and local time step dtl
   (src/solver/solverUtils.F90:43-355).  onlyRadii = 1 does nothing unless the residual of the level reads the radii
   (scalar dissipation: spaceDiscr up to the ground level, spaceDiscrCoarse above it), as in the reference; the radii
   are scaled directionally only up to the ground level and only with spaceDiscr = scalar dissipation (dirScaling). */
int adfb_timestep(int level, int onlyRadii);
/* `initres(1,nwf); sourceTerms; residual` as called by the smoothers
   (src/solver/smoothers.F90:73-75, src/solver/multiGrid.F90:883-888): block-path
   mean-flow residual_block (src/solver/residuals.F90:4-346) with
   rFil = cdisRK(rkStage+1); the dissipative+viscous part fw persists on the device. */
int adfb_smoother_residual(int level, int rkStage);
/* executeRkStage (src/solver/smoothers.F90:90-382), rkStage = 1..nRKStages */
int adfb_rk_stage(int level, int rkStage);
/* RungeKuttaSmoother (src/solver/smoothers.F90:4-86); residual and dtl must be current */
int adfb_rk_cycle(int level);
/* executeDADIStep (src/solver/smoothers.F90:425-693): dw *= -cfl*dtl*vol, computedwDADI
   (src/solver/residuals.F90:1062-1748: three line-implicit sweeps of 5 scalar tridiagonal
   systems), primitive update, BCs, halo exchange */
int adfb_dadi_step(int level);
/* turbSolveDDADI (src/turbulence/turbAPI.F90:4-95): nSubIterTurb x { sa_block(.false.) on every
   block = SA residual with its implicit diagonal, three diagonally dominant ADI sweeps
   (saSolve, src/turbulence/sa.F90:717-1267), nuTilde update + clip, eddy viscosity,
   turbulence BCs; whalo2(nt1, nt2, F, F, T) } */
int adfb_sa_ddadi(int level, int nSubIterTurb);
/* DADISmoother (src/solver/smoothers.F90:383-421) */
int adfb_dadi_cycle(int level, int nSubiterations);

/* ---- ANK pieces (module ANKSolver, src/NKSolver/NKSolvers.F90) -------------------------------------------------
   The approximate Newton-Krylov solver keeps PETSc's GMRES; the library provides the operator it applies and the
   two per-cell reductions around it.  State vectors hold nState = 5 (ANK_coupled = 0: flow variables only) or nw
   (coupled) entries per owned cell, cell-major like getStates (setWANK :2975-3011). */
typedef struct AdfbAnkParams {
    double cfl;             /* ANK_CFL */
    double cflLimit;        /* ANK_CFLLimit (blending of the characteristic time step) */
    double turbCFLScale;    /* ANK_turbCFLScale */
    double physLSTol;       /* ANK_physLSTol */
    double physLSTolTurb;   /* ANK_physLSTolTurb */
    double stepMin;         /* ANK_stepMin */
    double stepFactor;      /* ANK_stepFactor */
    double machInf;         /* inputPhysics mach (VLR / Turkel truncation) */
    int32_t coupled;        /* ANK_coupled: turbulence variable in the vectors */
    int32_t useDissApprox;  /* ANK_useDissApprox -> blocketteRes(useDissApprox) */
    int32_t useFullVisc;    /* ANK_useFullVisc: useViscApprox = (.not. useFullVisc) .and. useDissApprox (:2489) */
    int32_t charTimeStepType; /* ANK_charTimeStepType: 0 'None', 1 'VLR', 2 'Turkel' */
} AdfbAnkParams;
int adfb_ank_set_params(const AdfbAnkParams* ank);
/* computeTimeStepMat / computeTimeStepBlock (:2041-2329): the nState x nState block of every owned cell from the
   CURRENT state, dtl (last time-step evaluation) and ANK_CFL; kept on the device for adfb_ank_form_function */
int adfb_ank_time_step_mat(void);
/* FormFunction_mf of ANKSolver (:2468-2538): setWANK(inVec); blocketteRes(useDissApprox, useViscApprox, useTurbRes =
   coupled); setRVec / setRVecANK; rVec += timeStepMat * inVec */
int adfb_ank_form_function(const double* inVec, double* rVec, long long n);
/* matrix-free product with that function (the MatMFFD shell of the ANK KSP, :1890-1905): base state U (host), then
   y = (F(U + h a) - F(U)) / h for host vectors; h <= 0: PETSc's default differencing parameter as in adfb_mffd_apply */
int adfb_ank_mffd_set_base(const double* U, long long n);
int adfb_ank_mffd_apply(const double* a, double* y, long long n, double h);
/* Turbulence KSP of the decoupled ANK (ANKTurbSolveKSP, NKSolvers.F90:3337 ff.); vectors hold the nt1:nt2 = one turbulence
   variable per owned cell, cell order like getStates.
   adfb_ank_form_function_turb = FormFunction_mf_turb (:2540-2612): setWANK(inVec, nt1, nt2); blocketteRes(useFlowRes = .false.);
   setRVecANKTurb (dw(itu1) / volRef * turbResScale); + inVec / (ANK_CFL dtl volRef) * turbResScale / ANK_turbCFLScale.
   adfb_ank_mffd_turb_set_base / _apply: the MatMFFD shell over it, y = (F(U + h a) - F(U)) / h (h > 0 given by the caller).
   adfb_ank_physicality_check_turb = physicalityCheckANKTurb (:3212-3335): lambdaP MIN-reduced over all ranks, deltaW returned
   with the clipped updates. */
int adfb_ank_form_function_turb(const double* inVec, double* rVec, long long n);
int adfb_ank_mffd_turb_set_base(const double* U, long long n);
int adfb_ank_mffd_turb_apply(const double* a, double* y, long long n, double h);
int adfb_ank_physicality_check_turb(const double* wVec, double* deltaW, long long n, double* lambdaP);
/* the same product with a and y resident on this GPU (PETSc VECCUDA arrays): no PCIe traffic */
int adfb_ank_mffd_apply_device(const double* aDev, double* yDev, long long n, double h);
/* physicalityCheckANK (:3013-3210): largest step lambda <= *lambdaP that changes rho and rhoE by at most physLSTol
   (and decreases the turbulence variable by at most physLSTolTurb; individual turbulence updates that would be more
   limiting than stepFactor * stepMin are clipped in deltaW instead), MIN-reduced over the ranks */
int adfb_ank_physicality_check(const double* wVec, double* deltaW, long long n, double* lambdaP);

/* Device GMRES for the two matrix-free operators: what PETSc's KSPGMRES does for NK_KSP / ANK_KSP (NKSolvers.F90:395-435,
   2009-2037: restart = subspace, right preconditioning, classical Gram-Schmidt without refinement, zero initial guess),
   with the Krylov basis resident on the GPU.  op 0: the NK product (adfb_mffd_set_base first), op 1: the ANK product
   (adfb_ank_time_step_mat + adfb_ank_mffd_set_base first), op 2: the block-diagonal time-step matrix alone (a linear
   operator; used to verify the solver).  pc == NULL: identity; otherwise pc(ctx, inDev, outDev, n) applies
   the right preconditioner M^-1 to a DEVICE vector (the reference's ASM/ILU of the assembled approximate Jacobian stays
   with PETSc).  rhs, x: host vectors; its / resNorm (||b - A x|| estimate) may be NULL. */
typedef int (*AdfbPrecondFn)(void* ctx, const double* inDev, double* outDev, long long n);
int adfb_gmres_solve(int op, const double* rhs, double* x, long long n, int restart, int maxIts, double rtol, double atol,
                     AdfbPrecondFn pc, void* pcCtx, int* its, double* resNorm);

/* ---- multigrid (src/solver/multiGrid.F90) ------------------------------------------------------------------
   Grid levels: blocks created with level = 1 (finest) .. n; geometry, BCs and the communication pattern are set
   per block / per level like on the finest level (coarse levels exchange the first halos only: pass the 1st-halo
   lists, commPatternCell_1st / internalCell_1st).  On levels > 1 the entry points take the reference's
   currentLevel > groundLevel branches: dw starts from the residual forcing term wr (initRes_block,
   residuals.F90:485-497), first-order scalar dissipation with vis2Coarse (inviscidDissFluxScalarCoarse,
   fluxes.F90:4977-5203, or inviscidDissFluxMatrixCoarse :5205-5711 with spaceDiscrCoarse = ADFB_DISS_MATRIX), no directional scaling of the spectral radii
   (solverUtils.F90:106), cflCoarse and no second halos in the RK stage (smoothers.F90:131-140), constant-pressure
   walls (BCRoutines.F90:550,642,1100), frozen eddy viscosity (turbUtils.F90:606-616).
   adfb_block_set_mg: tables of createCoarseBlocks (src/preprocessing/coarseUtils.F90:254-420) with the reference's
   extents: mg{I,J,K}Fine(1:ie,2), mg{I,J,K}Weight(2:il) of the COARSE block, mg{I,J,K}Coarse(2:il,2) of the FINE block. */
int adfb_block_set_mg(int coarseBlk, int fineBlk, const int32_t* mgIFine, const int32_t* mgJFine, const int32_t* mgKFine,
                      const double* mgIWeight, const double* mgJWeight, const double* mgKWeight, const int32_t* mgICoarse,
                      const int32_t* mgJCoarse, const int32_t* mgKCoarse);
/* transferToCoarseGrid (multiGrid.F90:5-324) from fineLevel to fineLevel + 1: fine residual, restriction of the
   solution (volume weighted) and of the residual, setCornerRowHalos, applyAllBC(.false.), whalo1, timeStep, w1/p1,
   coarse residual and the residual forcing term wr (relaxation fcoll) */
int adfb_mg_restrict(int fineLevel);
/* transferToFineGrid(corrections = .true.) (multiGrid.F90:326-654) from fineLevel + 1 to fineLevel: corrections
   w - w1 / p - p1, setCorrectionsCoarseHalos (mgBoundCorr), trilinear interpolation, state update, BCs, exchange */
int adfb_mg_prolong(int fineLevel);
/* Full-multigrid start-up, the solver loop `do groundLevel = mgStartlevel, 1, -1` (src/solver/solvers.F90:63-117):
   adfb_set_ground_level = iteration%groundLevel, the finest level of the cycles that follow (levels above it take the
   coarse-level branches; a coarse ground level runs the fine-grid routines with cflCoarse and second halos, and needs
   second-level halo lists for that level).  Any pair of spaceDiscr and spaceDiscrCoarse: on a coarse ground level
   adfb_residual (blocketteRes) uses spaceDiscr, the smoother and multigrid entry points the fine-grid routines of
   spaceDiscrCoarse (residual_block with currentLevel /= 1);
   adfb_mg_prolong_solution = transferToFineGrid(corrections = .false.) (multiGrid.F90:326-654) with extrapolateSolution
   (:656-737) and extrapolateViscosities (:739-823): the solution of ground level fineLevel + 1 interpolated to fineLevel,
   halos extrapolated, turbulence + flow BCs and the exchanges as the reference orders them.  Lower the ground level
   afterwards. */
int adfb_set_ground_level(int level);
int adfb_get_ground_level(void);
int adfb_mg_prolong_solution(int fineLevel);
/* executeMGCycle (multiGrid.F90:825-955) on the ground level (adfb_set_ground_level, default 1) with the strategy of setCycleStrategy (:957-1030):
   cycling(1:nSteps) in {-1 prolongate, 0 smooth, +1 restrict}; smoother 0 = RungeKuttaSmoother, n >= 1 = DADISmoother
   with nSubiterations = n (smoothers.F90:400-420).  Ends like the reference
   with turbSolveDDADI (RANS), timeStep and the ground-level residual. */
int adfb_mg_cycle(int nSteps, const int* cycling, int smoother);

#ifdef __cplusplus
}
#endif
#endif /* ADFLOW_B200_H */
