"""The reference's own infChangeCorrection and setUniformFlow (src/initFlow/initializeFlow.F90:191-316, :2143-2286) and
getRotMatrix / myNorm2 (src/utils/utils.F90:6591-6665, :1696-1702), translated Fortran -> C with oracle/f90toc.py where the
reference source lies, compiled into a temporary directory and linked against oracle/_ref/libblockette_ref.so, whose
module variables, blockPointers, BCData and translated BC routines they share (oracle/refblockette.py binds them).
Test infrastructure only: nothing is written into the tree; without the reference or oracle/_ref, available() is False.

Source patches (none on the arithmetic of the path; the translator's own list, PATCHES of oracle/make_ref.py, applies
except its two rotating-frame `rotmatrix` rules, which would rename getRotMatrix):
- adjustInflowAngle / referenceState -> no-ops: the harness sets wInf, as adfb_set_params does on the device
- the character dummy correctionType -> an integer flag: "offset" = 0, "rotate" = 1 (the device's `type`)
- setUniformFlow's time-spectral internal-flow branch (:2213-2286, with its mpi_allreduce) dropped: not built
- matmul(rotMat, vCell) -> rotMat(:, 1) * vCell(1) + rotMat(:, 2) * vCell(2) + rotMat(:, 3) * vCell(3), and
  Wmat2 = matmul(Wmat, Wmat) -> ank_matmul (oracle/ref_env.c): gfortran's inline matmul, a sum from zero in index order;
  vec3 = vec3 / sqrt(sum(vec3**2)) -> f90_normalize3 below: the norm is formed once before the assignment, as Fortran's
  array assignment requires (the translator would re-form it from the updated elements), with gfortran's inline sum
- the function myNorm2 -> a subroutine with the result as last dummy (the translator handles subroutines only); a
  two-line C adaptor below gives its callers the function back
- oversetPresent is the harness global `oversetpresent`; mgStartLevel is defined here
whalo2 is the single-block whalo2 of the reference: no neighbours and no orphans, so only its closing
computeEtotBlock(2, il, 2, jl, 2, kl) (haloExchange.F90:174-197), through the translated computeEtotBlock."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
_REFDIR = os.path.join(ROOT, "oracle", "_ref")
_SO_BASE = os.path.join(_REFDIR, "libblockette_ref.so")

_SHIM = r"""
#include <math.h>
#include "ref_env.h"
#include "ref_protos.h"
int mgstartlevel = 1;
void utils_mynorm2s(double* x, double* r);
double mynorm2(double* x) { double r; utils_mynorm2s(x, &r); return r; }
void f90_normalize3(double* v) {
    const double s = sqrt((v[0] * v[0] + v[1] * v[1]) + v[2] * v[2]);
    for (int i = 0; i < 3; i++) v[i] = v[i] / s;
}
/* whalo2 on one block without neighbours or orphans: the closing computeEtotBlock on the owned cells */
void whalo2(int* level, int* start, int* end, int* commpressure, int* commgamma, int* commviscous) {
    (void)level; (void)commgamma; (void)commviscous;
    if (*commpressure && *start <= 5 && *end >= 5) {
        int two = 2, cfk = getcorrectfork();
        flowutils_computeetotblock(&two, &bp_il, &two, &bp_jl, &two, &bp_kl, &cfk);
    }
}
"""

_L = None


def available():
    return os.path.exists(os.path.join(REF, "src", "initFlow", "initializeFlow.F90")) and os.path.exists(_SO_BASE)


def _translate(outdir):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import f90toc
    import make_ref as M

    env = f90toc.Env(M.ENV_INTS + ["mgstartlevel", "flowtype", "internalflow"], M.env_arrays(),
                     ["getcorrectfork", "bcd_icbeg", "bcd_icend", "bcd_jcbeg", "bcd_jcend", "bcd_inbeg", "bcd_inend", "bcd_jnbeg",
                      "bcd_jnend", "bcd_iblank", "bcd_subsonicinlettreatment", "cbcd_icbeg", "cbcd_icend", "cbcd_jcbeg", "cbcd_jcend"],
                     dict(M.ENV_SUBS, getrotmatrix=[("vec1", "double", True), ("vec2", "double", True), ("rotmat", "double", True)],
                          f90_normalize3=[("v", "double", True)]))
    base = [p for p in M.PATCHES if "rotmatrix" not in p[0]]
    init_patches = [
        (r"^call adjustinflowangle\(\)$", "continue"),
        (r"^call referencestate$", "continue"),
        (r"^character\*\(\*\), intent\(in\) :: correctiontype$", "integer(kind=inttype), intent(in) :: correctiontype"),
        (r'^if \(correctiontype \.eq\. "offset"\) then$', "if (correctiontype == 0) then"),
        (r'^else if \(correctiontype \.eq\. "rotate"\) then$', "else if (correctiontype == 1) then"),
        (r"matmul\(rotmat, vcell\)", "rotmat(:, 1) * vcell(1) + rotmat(:, 2) * vcell(2) + rotmat(:, 3) * vcell(3)"),
        ("block", r"^testcorrection: if", r"^end if testcorrection"),
    ] + base
    utils_patches = [
        (r"^function mynorm2\(x\)$", "subroutine mynorm2s(x, mynorm2)"),
        (r"^real\(kind=realtype\) :: mynorm2$", "real(kind=realtype), intent(out) :: mynorm2"),
        (r"^end function mynorm2$", "end subroutine mynorm2s"),
        (r"^wmat2 = matmul\(wmat, wmat\)$", "call ank_matmul(wmat, wmat, wmat2)"),
        (r"^vec3 = vec3 / sqrt\(sum\(vec3\*\*2\)\)$", "call f90_normalize3(vec3)"),
    ] + base
    out = []
    tr = None
    for rel, prefix, only, patches in (("initFlow/initializeFlow.F90", "initializeflow_", {"infchangecorrection", "setuniformflow"},
                                        init_patches),
                                       ("utils/utils.F90", "utils_", {"getrotmatrix", "mynorm2s"}, utils_patches)):
        code, tr = f90toc.translate_module(os.path.join(REF, "src", rel), only=only, env=env, rename_modules=M.RENAME_MODULES,
                                           patches=patches, defined=(), tr=tr, prefix=prefix)
        path = os.path.join(outdir, os.path.basename(rel).replace(".F90", "").lower() + "_infchange.c")
        with open(path, "w") as f:
            f.write(code)
        out.append(path)
    # getRotMatrix is called unprefixed from initializeFlow (module utils): the translated one carries the prefix
    decl = ('#include "ref_protos.h"\nextern int mgstartlevel;\ndouble mynorm2(double* x);\nvoid f90_normalize3(double* v);\n'
            "void utils_getrotmatrix(double* vec1, double* vec2, double* rotmat);\n")
    for q, path in enumerate(out):
        with open(path) as f:
            code = f.read()
        if q == 0:
            code = code.replace("getrotmatrix(", "utils_getrotmatrix(")
        with open(path, "w") as f:
            f.write(code.replace('#include "ref_protos.h"\n', decl, 1))
    with open(os.path.join(outdir, "shim_infchange.c"), "w") as f:
        f.write(_SHIM)
    return out + [os.path.join(outdir, "shim_infchange.c")]


def lib():
    """the compiled translation (built once per source state into the temporary directory)"""
    global _L
    if _L is not None:
        return _L
    from oracle import refblockette as rb

    rb.lib()   # the shared library of the module variables first, so that both see one copy
    h = hashlib.sha1()
    for p in (__file__, os.path.join(ROOT, "oracle", "f90toc.py"), os.path.join(ROOT, "oracle", "make_ref.py"),
              os.path.join(REF, "src", "initFlow", "initializeFlow.F90"), os.path.join(REF, "src", "utils", "utils.F90"), _SO_BASE):
        with open(p, "rb") as f:
            h.update(f.read())
    # the library is bound to this tree's libblockette_ref.so by its run path: a checkout elsewhere with the same sources
    # must not load it, or the translation and the harness would each see their own copy of the module variables
    h.update(os.path.abspath(_SO_BASE).encode())
    outdir = os.path.join(tempfile.gettempdir(), "adfb_ref_infchange_%d_%s" % (os.getuid(), h.hexdigest()[:12]))
    so = os.path.join(outdir, "libinfchange_ref.so")
    if not os.path.exists(so):
        os.makedirs(outdir, exist_ok=True)
        # sources and library in a directory of this process's own: test processes running side by side may build at once
        work = tempfile.mkdtemp(dir=outdir)
        try:
            srcs = _translate(work)
            tmp = os.path.join(work, "libinfchange_ref.so")
            subprocess.check_call(["gcc", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-std=gnu11", "-w", "-shared",
                                   "-I" + _REFDIR, "-I" + os.path.join(ROOT, "oracle"), "-Wl,-Bsymbolic", "-o", tmp] + srcs
                                  + [_SO_BASE, "-Wl,-rpath," + _REFDIR, "-lm"])
            os.replace(tmp, so)
        finally:
            shutil.rmtree(work, ignore_errors=True)
    _L = C.CDLL(so)
    return _L


def _bind(hb, prm, overset=False, mg_start=1):
    from oracle import refblockette as rb

    rb.set_params(prm, hb.nw)
    C.c_void_p.in_dll(rb.lib(), "setpointers_hook").value = None   # setPointers: the one bound block
    rb._seti("anksolver_nstate", 3)   # ank_matmul's dimension: the 3 x 3 of getRotMatrix
    rb._seti("oversetpresent", int(overset))
    rb._seti("bp_ndom", 1)
    C.c_int.in_dll(lib(), "mgstartlevel").value = mg_start
    blk = rb.RefBlock(hb, prm)
    blk.bind()
    blk.keep = rb.bind_bcs(hb, prm)
    rb._BOUND = blk
    return blk


def _copy_back(blk, hb):
    import numpy as np

    for ref, mine in (("w", "w"), ("p", "p"), ("rlv", "rlv"), ("rev", "rev"), ("dw", "dw"), ("fw", "fw")):
        np.copyto(getattr(hb, mine), blk.a[ref])


def inf_change_correction(hb, prm, old_winf, tol=1e-12, kind="offset", overset=False):
    """the translated infChangeCorrection on one level-1 block (in place); prm holds the new free stream"""
    blk = _bind(hb, prm, overset)
    old = (C.c_double * 5)(*[float(v) for v in list(old_winf)[:5]])
    lib().initializeflow_infchangecorrection(old, C.byref(C.c_double(tol)), C.byref(C.c_int({"offset": 0, "rotate": 1}[kind])))
    _copy_back(blk, hb)


def set_uniform_flow(hb, prm, mu_inf, eddy_vis_inf_ratio, level=1):
    """the translated setUniformFlow with mgStartLevel = level on hb bound as that level's block (in place)"""
    from oracle import refblockette as rb

    blk = _bind(hb, prm, mg_start=level)
    rb._setd("muinf", mu_inf)
    rb._setd("eddyvisinfratio", eddy_vis_inf_ratio)
    lib().initializeflow_setuniformflow()
    _copy_back(blk, hb)


def rot_matrix(vec1, vec2):
    """the translated getRotMatrix; rotMat as a 3 x 3 nested list rotMat(i, j) -> [i - 1][j - 1]"""
    from oracle import refblockette as rb

    lib()
    rb._seti("anksolver_nstate", 3)
    a = (C.c_double * 3)(*vec1)
    b = (C.c_double * 3)(*vec2)
    r = (C.c_double * 9)()
    lib().utils_getrotmatrix(a, b, r)
    return [[r[i + 3 * j] for j in range(3)] for i in range(3)]
