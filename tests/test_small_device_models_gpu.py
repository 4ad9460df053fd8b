"""The GPU parity files under ADFB_SM_COUNT=1 and 5: the launch choosers plan for a device of that many multiprocessors.

ftile_choose (k_flowres), sa_tile_choose (k_sa) and lines_per_cta (k_resavg_lines) size their k chunks and line counts
from the device's SM count, so on an H100 the small blocks of the suite get configurations the production blocks never
do: one or two k planes per CTA, a handful of lines per CTA.  With one SM the tile kernels march whole blocks and the
residual averaging puts as many lines into a CTA as its shared memory holds; with five the chunks are several and of
uneven length.  Every pick is a legal launch (no kernel relies on co-resident CTAs), so every parity test must pass as it
does with the device's own count.  A second run of three tests under the kernel trace shows that the long chunks and
line tables did run."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FILES = ["test_residual_parity.py", "test_cuda_vs_reference.py", "test_smoother_parity.py", "test_regimes_gpu.py", "test_dadi.py",
         "test_sa_solve.py", "test_form_function_pipeline.py", "test_mffd.py", "test_diss_continuation_gpu.py",
         "test_multiblock_vectors.py", "test_mg_gpu.py", "test_ank_gpu.py"]
# tests whose launches show the configurations: the 5 x 6 x 40 block (one k_sa tile of 16 x 8, 40 planes) and the
# 36 x 19 x 41 block of residual averaging (684 lines in its shortest direction)
SA_NODE = "tests/test_residual_parity.py::test_rans_sa_residual_matches_oracle[shape2]"
RA_NODE = "tests/test_smoother_parity.py::test_residual_averaging_matches_oracle[shape2]"
SA_PLANES, RA_FEWEST_LINES = 40, 36 * 19


def _env(n_sm, **kw):
    e = dict(os.environ, ADFB_SM_COUNT=str(n_sm), **kw)
    for k in ("ADFB_SA_TILE", "ADFB_TILE"):
        e.pop(k, None)
    e["PYTHONPATH"] = os.pathsep.join([HERE] + ([e["PYTHONPATH"]] if e.get("PYTHONPATH") else []))
    return e


def _pytest(args, env, timeout):
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", "--rootdir", ROOT] + args, cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]


@pytest.mark.parametrize("n_sm", [1, 5])
def test_parity_files_pass(cuda_lib, n_sm):
    _pytest([os.path.join(HERE, f) for f in FILES] + ["-m", "gpu", "-x"], _env(n_sm), 3000)


@pytest.mark.parametrize("n_sm", [1, 5])
def test_long_chunks_and_line_tables_ran(cuda_lib, n_sm, tmp_path):
    """from the grid / block args of the Kineto trace: k_sa with fewer k chunks than planes, k_flowres with chunks longer
    than two planes, k_resavg_lines with more than 12 lines per CTA"""
    out = tmp_path / "launches.json"
    _pytest(["-p", "kernel_trace", "--kernel-launches", str(out), SA_NODE, RA_NODE], _env(n_sm, ADFB_NO_GRAPH="1"), 900)
    with open(out) as f:
        seen = json.load(f)

    def launches(node, name):
        got = [(g, b) for n, g, b in seen[node] if n == name or n.startswith(name + "<")]
        assert got and all(g is not None for g, _ in got), "%s: no %s launch with a grid in the trace" % (node, name)
        return got

    assert any(g[2] < SA_PLANES for g, _ in launches(SA_NODE, "k_sa")), launches(SA_NODE, "k_sa")
    assert any(-(-SA_PLANES // g[2]) > 2 for g, _ in launches(SA_NODE, "k_flowres")), launches(SA_NODE, "k_flowres")
    assert any(g[0] * 12 < RA_FEWEST_LINES for g, _ in launches(RA_NODE, "k_resavg_lines")), launches(RA_NODE, "k_resavg_lines")
