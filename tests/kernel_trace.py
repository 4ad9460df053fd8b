"""pytest plugin: record which of the library's kernels each test launches.

Load it with ``-p kernel_trace`` (``tests`` on PYTHONPATH) and ``--kernel-trace=OUT.json``.  Every test call runs under
torch.profiler with CUDA activity; the kernel names of the trace are put in canonical form (kernel_table.canonical) and
written as ``{nodeid: [kernels]}``.  With ``--kernel-launches=OUT.json`` the launch configurations are written as well,
``{nodeid: [[kernel, grid, block], ...]}`` (each distinct configuration once), from the ``grid`` / ``block`` args of the
kernel events of the Kineto trace.  Kernels replayed from a CUDA graph may not be reported one by one, so the runs that
use this plugin set ADFB_NO_GRAPH=1."""
import json
import os
import tempfile

import pytest

from kernel_table import canonical

_seen = {}
_launches = {}


def pytest_addoption(parser):
    parser.addoption("--kernel-trace", action="store", default=None, help="write {nodeid: [canonical kernel names]} here")
    parser.addoption("--kernel-launches", action="store", default=None, help="write {nodeid: [[kernel, grid, block], ...]} here")


def launches(prof):
    """[(canonical kernel, grid, block)] of this library's kernel launches in a finished torch.profiler run (distinct
    configurations, sorted); grid / block are None where the trace has no such arg"""
    fd, path = tempfile.mkstemp(suffix=".json")
    os.close(fd)
    try:
        prof.export_chrome_trace(path)
        with open(path) as f:
            trace = json.load(f)
    finally:
        os.unlink(path)
    out = set()
    for e in trace.get("traceEvents", []):
        if e.get("cat") != "kernel":
            continue
        n = canonical(e.get("name", ""))
        if n is None:
            continue
        a = e.get("args", {})
        g, b = a.get("grid"), a.get("block")
        out.add((n, None if g is None else tuple(g), None if b is None else tuple(b)))
    return sorted(out, key=repr)


@pytest.hookimpl(hookwrapper=True)
def pytest_runtest_call(item):
    if not (item.config.getoption("--kernel-trace") or item.config.getoption("--kernel-launches")):
        yield
        return
    import torch
    from torch.profiler import ProfilerActivity, profile

    gpu = torch.cuda.is_available()
    if gpu:
        torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU] + ([ProfilerActivity.CUDA] if gpu else [])) as prof:
        yield
        if gpu:
            torch.cuda.synchronize()
    names = {canonical(e.name) for e in prof.events()}
    names.discard(None)
    _seen[item.nodeid] = sorted(names)
    if item.config.getoption("--kernel-launches"):
        _launches[item.nodeid] = [list(x) for x in launches(prof)]


def pytest_sessionfinish(session):
    for opt, rec in (("--kernel-trace", _seen), ("--kernel-launches", _launches)):
        out = session.config.getoption(opt)
        if out:
            with open(out, "w") as f:
                json.dump(rec, f, indent=1, sort_keys=True)
