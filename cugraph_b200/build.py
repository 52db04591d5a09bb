"""Build cugraph_b200/lib/libcugraph_c.so (the C-ABI boundary) with nvcc for sm_90a (H100).

In-tree, incremental (per-file objects under cugraph_b200/csrc/_obj), parallel.  The .so is
git-ignored.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(CSRC, "_obj")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libcugraph_c.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "--expt-relaxed-constexpr", "-Xcompiler", "-fPIC,-fvisibility=hidden",
         "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-ccbin", "/usr/bin/g++"] + os.environ.get("B200_EXTRA_NVCC_FLAGS", "").split()


def _newer(a, b):
    return (not os.path.exists(b)) or os.path.getmtime(a) > os.path.getmtime(b)


def _headers_mtime():
    m = 0.0
    for d in (CSRC, os.path.join(ROOT, "include", "cugraph_c")):
        for f in os.listdir(d):
            if f.endswith((".cuh", ".h", ".hpp")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    return m


def _compile(src, obj, verbose):
    cmd = [NVCC] + ARCH + FLAGS + ["-c", src, "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    return src, r.returncode, r.stdout + r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    srcs = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    hm = _headers_mtime()
    jobs = []
    objs = []
    for f in srcs:
        src = os.path.join(CSRC, f)
        obj = os.path.join(OBJ, f[:-3] + ".o")
        objs.append(obj)
        if force or _newer(src, obj) or hm > os.path.getmtime(obj):
            jobs.append((src, obj))
    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            for src, rc, out in ex.map(lambda j: _compile(j[0], j[1], verbose), jobs):
                if verbose or rc != 0:
                    sys.stderr.write(out)
                if rc != 0:
                    raise RuntimeError(f"nvcc failed on {src}")
    if jobs or not os.path.exists(LIB) or any(_newer(o, LIB) for o in objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    _build_cbench(force or bool(jobs))
    return LIB


def _build_cbench(force):
    """scripts/cbench.cu -> cugraph_b200/lib/cbench: the Python-free development probe"""
    src = os.path.join(ROOT, "scripts", "cbench.cu")
    out = os.path.join(LIBDIR, "cbench")
    if not os.path.exists(src) or not (force or _newer(src, out) or _newer(LIB, out)):
        return
    cmd = [NVCC, "-O2", "-std=c++17"] + ARCH + ["-I", os.path.join(ROOT, "include"), src, "-o", out, "-L", LIBDIR,
                                                 "-l:libcugraph_c.so", "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN", "-ccbin", "/usr/bin/g++"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:  # a development tool: report, do not fail the library build
        sys.stderr.write("cbench not built:\n" + r.stdout + r.stderr)


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
