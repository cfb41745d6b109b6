"""Build libopenstereo_b200.so (sm_90a, H100) in-tree with nvcc.

    python -m openstereo_b200.build [--force] [--verbose]

The shared library is the whole native product: hand-written CUDA kernels behind the C ABI of
include/openstereo_b200.h.  It is built IN-TREE (openstereo_b200/lib/) so that the package imports
from the repository tree; nvcc cross-compiles without a GPU.
"""
import argparse
import glob
import hashlib
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libopenstereo_b200.so")
STAMP = os.path.join(LIBDIR, "build.stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found (looked on PATH and /usr/local/cuda/bin)")
    return cand


def _sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _fingerprint():
    h = hashlib.sha256()
    for path in _sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [
            os.path.join(ROOT, "include", "openstereo_b200.h"), os.path.abspath(__file__)]:
        with open(path, "rb") as f:
            h.update(os.path.relpath(path, ROOT).encode() + b"\0" + f.read())   # relative: the stamp survives a move of the tree
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every csrc/*.cu for sm_90a and link the shared library.  Returns its path."""
    os.makedirs(LIBDIR, exist_ok=True)
    fp = _fingerprint()
    if not force and os.path.exists(LIB) and os.path.exists(STAMP) and open(STAMP).read().strip() == fp:
        return LIB
    nvcc = _nvcc()
    objs = []
    logs = []
    procs = []
    for src in _sources():
        obj = os.path.join(LIBDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + NVCC_FLAGS + ["-I", os.path.join(ROOT, "include"), "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, proc in procs:
        out, _ = proc.communicate()
        logs.append("== %s\n%s" % (os.path.basename(src), out))
        if proc.returncode != 0:
            sys.stderr.write("\n".join(logs))
            raise RuntimeError("nvcc failed on %s" % src)
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-o", LIB] + objs
    res = subprocess.run(link, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout)
        raise RuntimeError("link failed")
    with open(os.path.join(LIBDIR, "ptxas.log"), "w") as f:
        f.write("\n".join(logs))
    with open(STAMP, "w") as f:
        f.write(fp)
    if verbose:
        print("\n".join(logs))
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose))
