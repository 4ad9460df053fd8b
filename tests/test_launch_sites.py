"""Every kernel launch of the library goes through one helper, launch_kernel (adflow_b200/csrc/adfb_common.cuh).

The helper puts each launch in its family's NVTX range, counts it once (adfb_launch_count, the per-family counts of
adfb_kernel_times and the per-graph counts of the graph cache) and sets the programmatic-dependent-launch attribute
when asked to.  On the CPU the sources are checked for launches that bypass it, and every kernel launched with the
attribute is checked to wait for its predecessor (ADFB_PDL_SYNC) before it touches memory: without that wait it would
race the kernel before it.  On the device the launch count of each entry point is held to the number of this library's
kernels that torch.profiler sees it launch."""
import json
import os
import re
import subprocess
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "adflow_b200", "csrc")
HELPER_FILE = "adfb_common.cuh"
HELPER_DEF = re.compile(r"static cudaError_t launch_kernel\(")


def _strip_comments(s):
    s = re.sub(r"/\*.*?\*/", " ", s, flags=re.S)
    return re.sub(r"//[^\n]*", "", s)


def _sources():
    return {f: _strip_comments(open(os.path.join(CSRC, f)).read()) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))}


def _closing(s, i, open_ch, close_ch):
    """index of the bracket that closes the one at s[i]"""
    depth = 0
    for j in range(i, len(s)):
        if s[j] == open_ch:
            depth += 1
        elif s[j] == close_ch:
            depth -= 1
            if depth == 0:
                return j
    raise AssertionError("unbalanced %s at %d" % (open_ch, i))


def _without_helper(src):
    """the helper file without the helper's own definition"""
    m = HELPER_DEF.search(src)
    assert m, "launch_kernel is not defined in %s" % HELPER_FILE
    b = src.index("{", m.end())
    return src[:m.start()] + src[_closing(src, b, "{", "}") + 1:]


def _split_args(s, n):
    """the first n top-level comma-separated arguments of s and the rest"""
    out, depth, start = [], 0, 0
    for j, c in enumerate(s):
        if c in "([{":
            depth += 1
        elif c in ")]}":
            depth -= 1
        elif c == "," and depth == 0:
            out.append(s[start:j].strip())
            start = j + 1
            if len(out) == n:
                return out, s[start:]
    raise AssertionError("fewer than %d arguments in launch_kernel(%s)" % (n + 1, s))


def launch_calls():
    """[(file, kernel, pdl)] of every launch_kernel call in the library's sources (kernel without template arguments)"""
    calls = []
    for f, src in _sources().items():
        if f == HELPER_FILE:
            src = _without_helper(src)
        for m in re.finditer(r"\blaunch_kernel\(", src):
            o = m.end() - 1
            (fam, pdl, _g, _b, _smem, _s), rest = _split_args(src[o + 1:_closing(src, o, "(", ")")], 6)
            assert re.fullmatch(r"K_[A-Z]+", fam), (f, fam)
            assert pdl in ("true", "false"), "%s: launch_kernel(%s, %s, ...): pdl must be a literal" % (f, fam, pdl)
            calls.append((f, re.match(r"\s*(\w+)", rest).group(1), pdl == "true"))
    return calls


def kernel_bodies():
    """{kernel: [bodies of its __global__ definitions]}"""
    bodies = {}
    for src in _sources().values():
        for m in re.finditer(r"__global__\s+void\s+(?:__\w+__\s*\([^)]*\)\s*)?(\w+)", src):
            b = src.index("{", m.end())
            bodies.setdefault(m.group(1), []).append(src[b:_closing(src, b, "{", "}") + 1])
    return bodies


def test_no_launch_bypasses_the_helper():
    bad = []
    for f, src in _sources().items():
        if f == HELPER_FILE:
            src = _without_helper(src)
        for tok in ("<<<", "cudaLaunchKernel", "cudaLaunchCooperativeKernel", "KT_BEGIN", "KT_END", "g_kt.begin", "g_kt.end"):
            if tok in src:
                bad.append((f, tok))
    assert not bad, "kernel launches or launch accounting outside launch_kernel: %s" % bad


def test_pdl_launches_wait_for_their_predecessor():
    calls = launch_calls()
    bodies = kernel_bodies()
    unknown = sorted({k for _, k, _ in calls if k not in bodies})
    assert not unknown, "launched kernels without a __global__ definition: %s" % unknown
    pdl = {k for _, k, p in calls if p}
    # the residual step's kernels run with the attribute; the list below is a floor, not the set
    assert {"k_prep", "k_flowres", "k_faces", "k_div", "k_dadi_thomas_tile", "k_resavg_lines"} <= pdl, sorted(pdl)
    racing = sorted(k for k in pdl if not all("ADFB_PDL_SYNC()" in b for b in bodies[k]))
    assert not racing, "launched with the PDL attribute but never wait for the predecessor: %s" % racing


# --------------------------------------------------------------------------------------------------------------------
# device: one count per kernel launched

def _traced_kernels(prof):
    """canonical names of this library's kernels in a finished torch.profiler run, one per launch"""
    from kernel_table import canonical

    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    try:
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    finally:
        os.unlink(path)
    names = (canonical(e.get("name", "")) for e in trace.get("traceEvents", []) if e.get("cat") == "kernel")
    return [n for n in names if n is not None]


def _measure(s, out, name, fn):
    import torch
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    c0 = s.launchCount()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out[name] = {"counted": s.launchCount() - c0, "traced": _traced_kernels(prof)}


def _run_entry_points(path):
    """runs the entry points with ADFB_NO_GRAPH=1 (every launch reported by itself) and writes what was counted and traced"""
    import numpy as np
    import torch

    from adflow_b200 import make_params
    from adflow_b200 import synthetic as syn
    from adflow_b200.solver import ADFLOW_B200, RES_FLOW, RES_TURB
    from test_mg_gpu import make_levels

    out = {}
    prm = make_params()
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(syn.make_block(24, 16, 16, prm))   # 16 planes: the page-locked form function runs as a slab pipeline
        _measure(s, out, "setParams", lambda: s.setParams(prm))
        _measure(s, out, "residual", lambda: s.residual(RES_FLOW | RES_TURB))
        s.applyBCs(True, True)
        s.timeStep(False)
        s.smootherResidual(0)
        _measure(s, out, "rkCycle", s.rkCycle)
        _measure(s, out, "dadiStep", s.dadiStep)
        U = s.getStates()
        s.mffdSetBase(U)
        b = np.random.default_rng(5).standard_normal(U.size) * np.abs(U).clip(1e-6) * 1e-3
        _measure(s, out, "gmresSolve", lambda: s.gmresSolve(b, "NK", restart=3, max_its=5, rtol=1e-12))
        n = U.size
        hw, hr = torch.empty(n, dtype=torch.float64).pin_memory(), torch.empty(n, dtype=torch.float64).pin_memory()
        hw.numpy()[:] = U
        _measure(s, out, "formFunction", lambda: s.formFunction(U))
        _measure(s, out, "formFunctionPtr", lambda: s.formFunctionPtr(hw.data_ptr(), hr.data_ptr(), n))
    finally:
        s.close()
    prm, levels = make_levels((16, 12, 8), None, 2)
    s = ADFLOW_B200(prm)
    try:
        s.addBlock(levels[0])
        s.addCoarseBlock(levels[1], 0)
        s.timeStep(False)
        s.smootherResidual(0)
        _measure(s, out, "mgCycle", lambda: s.mgCycle(ADFLOW_B200.cycleStrategy("2v")))
    finally:
        s.close()
    with open(path, "w") as f:
        json.dump(out, f, indent=1)


@pytest.mark.gpu
def test_launch_count_is_one_per_kernel(cuda_lib, tmp_path):
    out = tmp_path / "launches.json"
    e = dict(os.environ, ADFB_NO_GRAPH="1")
    e.pop("ADFB_FF_PIPE", None)
    e["PYTHONPATH"] = os.pathsep.join([ROOT, HERE] + ([e["PYTHONPATH"]] if e.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), str(out)], cwd=ROOT, env=e, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    with open(out) as f:
        got = json.load(f)
    assert sorted(got) == sorted(["setParams", "residual", "rkCycle", "dadiStep", "gmresSolve", "formFunction", "formFunctionPtr",
                                  "mgCycle"])
    for name, v in got.items():
        assert v["traced"], name
        assert v["counted"] == len(v["traced"]), (name, v["counted"], len(v["traced"]), sorted(set(v["traced"])))
    assert "k_param_consts" in got["setParams"]["traced"]
    assert {"k_axpy_many", "k_scale_to"} <= set(got["gmresSolve"]["traced"])
    # the page-locked call ran as the slab pipeline: another launch sequence than the pageable one
    assert got["formFunctionPtr"]["counted"] != got["formFunction"]["counted"]


if __name__ == "__main__":
    _run_entry_points(sys.argv[1])
