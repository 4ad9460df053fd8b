"""The kernel table (tests/kernel_table.py) lists exactly the library's kernel entry points, and every test it names exists.

A kernel added to the library without a test that reaches it, or a table row for a kernel the library no longer has,
fails here on the CPU; tests/test_dispatch_gpu.py checks on the device that the named tests really launch each kernel."""
import os
import re
import shutil
import subprocess
import sys

import pytest

from kernel_table import TABLE, canonical, excluded, reach

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
LIB = os.path.join(ROOT, "adflow_b200", "libadflow_b200.so")

# the only kernels no single-process test can launch: they fill and drain the buffers of a multi-rank halo exchange
ALLOWED_EXCLUSIONS = {"k_halo_pack", "k_halo_unpack", "k_halo_pack_interp"}


def _tool(name):
    p = shutil.which(name)
    if p:
        return p
    p = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)
    return p if os.path.exists(p) else None


def library_entries():
    """canonical names of the STO_ENTRY symbols of the library (cuobjdump -symbols, demangled by cu++filt)"""
    cuobjdump, filt = _tool("cuobjdump"), _tool("cu++filt")
    if not os.path.exists(LIB):
        pytest.skip("libadflow_b200.so not built")
    if not (cuobjdump and filt):
        pytest.skip("cuobjdump / cu++filt not found")
    out = subprocess.run([cuobjdump, "-symbols", LIB], capture_output=True, text=True, check=True).stdout
    mangled = [l.split()[-1] for l in out.splitlines() if "STO_ENTRY" in l]
    assert mangled, "no kernel entry points in %s" % LIB
    dem = subprocess.run([filt], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout.splitlines()
    assert len(dem) == len(mangled)
    names = [canonical(d) for d in dem]
    assert None not in names, [d for d, n in zip(dem, names) if n is None]
    assert len(set(names)) == len(names), "two entry points with one canonical name"
    return set(names)


def test_canonical_names():
    """the cu++filt spelling of the symbol table and the profiler's spelling give one canonical name"""
    assert canonical("void <unnamed>::k_faces<(bool)0, (bool)1, (int)2, (int)1, (bool)0, (int)0, (bool)0>(Dims, BlockDev, double, int, int)") \
        == "k_faces<0,1,2,1,0,0,0>"
    assert canonical("void (anonymous namespace)::k_faces<false, true, 2, 1, false, 0, false>(Dims, BlockDev, double, int, int)") \
        == "k_faces<0,1,2,1,0,0,0>"
    assert canonical("void <unnamed>::k_sa_thomas_part<(int)8, (int)12>(Dims, BlockDev, int, int, int, int, int, int, int)") == "k_sa_thomas_part<8,12>"
    assert canonical("<unnamed>::k_metrics(Dims, BlockDev, double)") == "k_metrics"
    assert canonical("(anonymous namespace)::k_metrics(Dims, BlockDev, double)") == "k_metrics"
    # kernels of other libraries (torch's own, cuBLAS) are not this library's
    assert canonical("void at::native::vectorized_elementwise_kernel<4, at::native::FillFunctor<double>>(int, double)") is None
    assert canonical("cudaLaunchKernel") is None


def test_table_matches_library_entry_points():
    lib = library_entries()
    missing, stale = sorted(lib - set(TABLE)), sorted(set(TABLE) - lib)
    assert not missing and not stale, "kernels without a table row: %s; table rows without a kernel: %s" % (missing, stale)


def test_table_rows_are_well_formed():
    for k, v in TABLE.items():
        assert canonical("<unnamed>::%s(" % k) == k, k
        assert isinstance(v, (reach, excluded)), k
        if isinstance(v, excluded):
            assert k in ALLOWED_EXCLUSIONS, "%s: not an allowed exclusion" % k
            assert v.reason
        else:
            assert v.node_ids, k
            assert all(re.fullmatch(r"ADFB_[A-Z0-9_]+", n) and isinstance(x, str) for n, x in v.env.items()), k


def test_table_node_ids_exist():
    ids = sorted({n for v in TABLE.values() if isinstance(v, reach) for n in v.node_ids})
    files = sorted({n.split("::")[0] for n in ids})
    r = subprocess.run([sys.executable, "-m", "pytest", "--collect-only", "-q", "-p", "no:cacheprovider", "--rootdir", ROOT] + files,
                       cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-2000:]
    collected = {l.strip() for l in r.stdout.splitlines() if "::" in l}
    unknown = [n for n in ids if n not in collected and not any(c.startswith(n + "[") for c in collected)]
    assert not unknown, "node ids that do not exist: %s" % unknown
