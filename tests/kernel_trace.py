"""pytest plugin: record which of the library's kernels each test launches.

Load it with ``-p kernel_trace`` (``tests`` on PYTHONPATH) and ``--kernel-trace=OUT.json``.  Every test call runs under
torch.profiler with CUDA activity; the kernel names of the trace are put in canonical form (kernel_table.canonical) and
written as ``{nodeid: [kernels]}``.  Kernels replayed from a CUDA graph may not be reported one by one, so the runs that
use this plugin set ADFB_NO_GRAPH=1."""
import json

import pytest

from kernel_table import canonical

_seen = {}


def pytest_addoption(parser):
    parser.addoption("--kernel-trace", action="store", default=None, help="write {nodeid: [canonical kernel names]} here")


@pytest.hookimpl(hookwrapper=True)
def pytest_runtest_call(item):
    if not item.config.getoption("--kernel-trace"):
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


def pytest_sessionfinish(session):
    out = session.config.getoption("--kernel-trace")
    if out:
        with open(out, "w") as f:
            json.dump(_seen, f, indent=1, sort_keys=True)
