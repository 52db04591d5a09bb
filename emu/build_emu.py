"""Build cugraph_b200/lib/libcugraph_c_emu.so: the single-GPU sources (staging, PageRank, BFS/SSSP) compiled as plain C++
against the host emulation shim in emu/ — test infrastructure for tests/test_emu_*_cpu.py."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "cugraph_b200", "csrc")
OUT = os.path.join(ROOT, "cugraph_b200", "lib", "libcugraph_c_emu.so")
SRCS = [os.path.join(CSRC, f) for f in ("capi_basic.cu", "capi_graph.cu", "graph_build.cu", "sweep_layout.cu", "sweep.cu", "pagerank.cu", "traverse.cu", "mg.cu", "generators.cu", "centrality.cu", "components.cu", "scc.cu", "graph_functions.cu")] + \
    [os.path.join(ROOT, "emu", "emu_debug.cpp")]


def build(force=False):
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    deps = SRCS + [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cuh")] + \
        [os.path.join(ROOT, "emu", f) for f in ("cuda_runtime.h", "cub/cub.cuh", "thrust/iterator/counting_iterator.h")]
    if not force and os.path.exists(OUT) and all(os.path.getmtime(d) <= os.path.getmtime(OUT) for d in deps):
        return OUT
    cmd = ["/usr/bin/g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-fvisibility=hidden", "-DB200_HOST_EMU",
           "-I", os.path.join(ROOT, "emu"), "-I", os.path.join(ROOT, "include"), "-I", CSRC, "-Wno-attributes"]
    for s in SRCS:
        cmd += ["-x", "c++", s]
    cmd += ["-o", OUT]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("emulation build failed")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv))
