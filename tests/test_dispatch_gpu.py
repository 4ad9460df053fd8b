"""Every kernel of the library is launched by the tests the kernel table names for it.

The tests of one environment (tests/kernel_table.py) run in one subprocess under the kernel_trace plugin, with
ADFB_NO_GRAPH=1 so that each launch is reported by itself; the run must pass, and each kernel of the group must appear in
the trace of one of its tests.  The switches that select a kernel (ADFB_FUSED, ADFB_SPLIT_FACES, ...) stay exercised
this way, and a change of the dispatch that leaves a kernel unreachable from its tests fails here."""
import json
import os
import subprocess
import sys

import pytest

from kernel_table import TABLE, reach

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def _groups():
    g = {}
    for k, v in TABLE.items():
        if isinstance(v, reach):
            g.setdefault(tuple(sorted(v.env.items())), {})[k] = v.node_ids
    return g


GROUPS = _groups()


@pytest.mark.parametrize("env", sorted(GROUPS), ids=lambda e: ",".join("%s=%s" % kv for kv in e) or "default")
def test_every_kernel_is_reached(cuda_lib, env, tmp_path):
    kernels = GROUPS[env]
    nodes = sorted({n for ids in kernels.values() for n in ids})
    out = tmp_path / "trace.json"
    e = dict(os.environ, ADFB_NO_GRAPH="1", **dict(env))
    e["PYTHONPATH"] = os.pathsep.join([HERE] + ([e["PYTHONPATH"]] if e.get("PYTHONPATH") else []))
    r = subprocess.run([sys.executable, "-m", "pytest", "-p", "kernel_trace", "--kernel-trace", str(out), "-q", "-p", "no:cacheprovider",
                        "--rootdir", ROOT] + nodes, cwd=ROOT, env=e, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    with open(out) as f:
        seen = json.load(f)
    for n in nodes:
        assert any(s == n or s.startswith(n + "[") for s in seen), "%s did not run" % n

    def traced(n):
        return set().union(*[set(v) for s, v in seen.items() if s == n or s.startswith(n + "[")])

    missing = {k: ids for k, ids in kernels.items() if not any(k in traced(n) for n in ids)}
    assert not missing, "kernels not launched by their tests: %s" % missing
