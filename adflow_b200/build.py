"""Build recipe for libadflow_b200.so (nvcc, sm_90a only, in-tree)."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libadflow_b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC", "-shared", "-Xptxas", "-v",
]


def sources():
    """everything the library depends on, this recipe included: a change of FLAGS (the target architecture) rebuilds it"""
    return [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh"))] + [
        os.path.join(HERE, "..", "include", "adflow_b200.h"), os.path.abspath(__file__)]


def stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(s) > t for s in sources())


def build(force=False, verbose=False):
    if not (force or stale()):
        return OUT
    cmd = [NVCC] + FLAGS + ["-o", OUT, os.path.join(CSRC, "adflow_b200.cu")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    log = os.path.join(HERE, "build.log")
    with open(log, "w") as f:
        f.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("nvcc failed, see %s" % log)
    if verbose:
        print(r.stderr)
    return OUT


if __name__ == "__main__":
    build(force="--force" in sys.argv, verbose=True)
