"""The monitor routines of convergenceInfo restated in numpy, in the reference's operation order, and the reference's own
maxHdiffMach / maxEddyv (src/utils/utils.F90:2422-2531) translated Fortran -> C with oracle/f90toc.py where the reference
source lies, compiled into a temporary directory and linked against oracle/_ref/libblockette_ref.so (whose translated
sumResiduals / sumAllResiduals, module variables and blockPointers they share, as tests/ref_inf_change.py does).
Test infrastructure only: nothing is written into the tree; without the reference or oracle/_ref, available() is False.

Source patch: `if (.not. monMachOrHMax) return` -> continue (the module flag monitor%monMachOrHMax is not part of the
harness; convergenceInfo calls maxHdiffMach for its values only when hdiff or mach is monitored).

The restatement (monitor_sums) gives adfb_monitor's out[10] for a list of HostBlocks: the sums accumulate cell by cell in
the reference's loop order (k, j, i; blocks in order) through np.cumsum, which adds sequentially; the maxima are the
largest cell values, formed with the reference's expression order."""
import ctypes as C
import hashlib
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
_REFDIR = os.path.join(ROOT, "oracle", "_ref")
_SO_BASE = os.path.join(_REFDIR, "libblockette_ref.so")
RANS = 3


def _seq_sum(start, terms):
    """start + t0 + t1 + ... added one by one, as a Fortran accumulation loop does"""
    return float(np.cumsum(np.concatenate(([start], terms)))[-1])


def _owned_f(a):
    """the values of an owned-cell array in Fortran order (i fastest)"""
    return np.asarray(a).ravel(order="F")


def monitor_sums(blocks, prm, what=3):
    """adfb_monitor's out[10] for the blocks `blocks` (HostBlocks with dw, vol, w, p, rlv, rev): sumResiduals for the
    variables 1..6, sumAllResiduals, hdiffMax, MachMax, eddyvisMax"""
    out = np.zeros(10)
    if what & 1:
        for hb in blocks:
            ow = hb.d.owned()
            vol = hb.vol[ow]
            for l in range(hb.nw):
                r = hb.dw[ow + (l,)] / vol                      # (dw / vol)**2
                out[l] = _seq_sum(out[l], _owned_f(r * r))
            ovv = 1.0 / vol
            state = np.zeros_like(vol)
            for l in range(hb.nw):
                t = hb.dw[ow + (l,)] * ovv
                if l >= 5:
                    t = t * prm.turbResScale                  # dw * ovv * turbResScale(l - nt1 + 1)
                state = state + t * t
            out[6] = _seq_sum(out[6], _owned_f(state))
    if what & 2:
        hinf = (prm.wInf[4] + prm.pInfCorr) / prm.rhoInf
        hmax = mmax = emax = 0.0
        for hb in blocks:
            ow = hb.d.owned()
            w, p = hb.w[ow], hb.p[ow]
            hdiff = np.abs((w[..., 4] + p) / w[..., 0] - hinf)
            mach2 = (w[..., 1] * w[..., 1] + w[..., 2] * w[..., 2] + w[..., 3] * w[..., 3]) * w[..., 0] / (prm.gammaInf * p)
            hmax = max(hmax, float(hdiff.max()))
            mmax = max(mmax, float(mach2.max()))
            if prm.equations == RANS:
                emax = max(emax, float((hb.rev[ow] / hb.rlv[ow]).max()))
        out[7], out[8], out[9] = hmax / hinf, float(np.sqrt(mmax)), emax
    return out


# ---------------------------------------------------------------------------------------------------------------------
# the reference's own routines
_L = None


def available():
    return os.path.exists(os.path.join(REF, "src", "utils", "utils.F90")) and os.path.exists(_SO_BASE)


def _translate(outdir):
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import f90toc
    import make_ref as M

    env = f90toc.Env(M.ENV_INTS, M.env_arrays(), ["getcorrectfork"], dict(M.ENV_SUBS))
    patches = [(r"^if \(\.not\. monmachorhmax\) return$", "continue")] + list(M.PATCHES)
    code, _ = f90toc.translate_module(os.path.join(REF, "src", "utils", "utils.F90"), only={"maxhdiffmach", "maxeddyv"}, env=env,
                                      rename_modules=M.RENAME_MODULES, patches=patches, defined=(), tr=None, prefix="monref_")
    path = os.path.join(outdir, "utils_monitor.c")
    with open(path, "w") as f:
        f.write(code)
    return [path]


def lib():
    """the compiled translation (built once per source state into the temporary directory)"""
    global _L
    if _L is not None:
        return _L
    from oracle import refblockette as rb

    rb.lib()
    h = hashlib.sha1()
    for p in (__file__, os.path.join(ROOT, "oracle", "f90toc.py"), os.path.join(ROOT, "oracle", "make_ref.py"),
              os.path.join(REF, "src", "utils", "utils.F90"), _SO_BASE):
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(os.path.abspath(_SO_BASE).encode())
    outdir = os.path.join(tempfile.gettempdir(), "adfb_ref_monitor_%d_%s" % (os.getuid(), h.hexdigest()[:12]))
    so = os.path.join(outdir, "libmonitor_ref.so")
    if not os.path.exists(so):
        os.makedirs(outdir, exist_ok=True)
        work = tempfile.mkdtemp(dir=outdir)
        try:
            srcs = _translate(work)
            tmp = os.path.join(work, "libmonitor_ref.so")
            subprocess.check_call(["gcc", "-O2", "-fno-fast-math", "-ffp-contract=off", "-fPIC", "-std=gnu11", "-w", "-shared",
                                   "-I" + _REFDIR, "-I" + os.path.join(ROOT, "oracle"), "-Wl,-Bsymbolic", "-o", tmp] + srcs
                                  + [_SO_BASE, "-Wl,-rpath," + _REFDIR, "-lm"])
            os.replace(tmp, so)
        finally:
            shutil.rmtree(work, ignore_errors=True)
    _L = C.CDLL(so)
    return _L


def reference_monitor(blocks, prm):
    """out[10] from the reference's sumResiduals, sumAllResiduals, maxHdiffMach and maxEddyv, block by block, combined as
    convergenceInfo does (monLoc: + for the sums, max for the maxima)"""
    from oracle import refblockette as rb

    L = lib()
    mon = (C.c_double * 16).in_dll(rb.lib(), "monloc")
    for q in range(16):
        mon[q] = 0.0
    maxima = [0.0, 0.0, 0.0]
    for hb in blocks:
        rb.call(hb, prm, "sumresiduals", 1, 1)
        for l in range(2, hb.nw + 1):
            rb.again("sumresiduals", l, l)
        rb.again("sumallresiduals", 7)
        rb._seti("eddymodel", int(prm.equations == RANS))
        hd, ma, ed = C.c_double(), C.c_double(), C.c_double()
        L.monref_maxhdiffmach(C.byref(hd), C.byref(ma))
        L.monref_maxeddyv(C.byref(ed))
        maxima = [max(maxima[0], hd.value), max(maxima[1], ma.value), max(maxima[2], ed.value)]
    mon = (C.c_double * 16).in_dll(rb.lib(), "monloc")
    return np.array([mon[q] for q in range(7)] + maxima)
