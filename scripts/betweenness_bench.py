"""Betweenness centrality (cugraph_betweenness_centrality) on symmetrised RMAT graphs, sampled and exact.

    python scripts/betweenness_bench.py [--scales 20 24] [--ks 64 256 1024] [--exact-scale 16] [--repeats 2]

For each scale, one graph (RMAT, edge factor 16, both directions of every edge) and, for each k, k sources drawn with
cugraph_select_random_vertices (seed 0): one warm-up call, then --repeats timed calls of the vertex betweenness (host
clock around the synchronous C-ABI call).  A last call with CUGRAPH_B200_BC_TRACE set gives every batch's time split into
BFS levels, sigma pull and backward pass (CUDA events, printed by the library to stderr and parsed here).  Traversed edges
per second = k * E / t, E = directed edges.  --exact-scale: every vertex a source.  One JSON line per run, with the card's
name and power limit read in the same process."""
import argparse
import json
import os
import re
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        return {"gpu_query_error": r.stderr.strip()[:200]}
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"card": name, "power_limit_w": float(power), "max_sm_clock_mhz": float(clock)}


def traced(fn):
    """(result, stderr text) of fn() with file descriptor 2 sent to a temporary file"""
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as f:
        os.dup2(f.fileno(), 2)
        try:
            out = fn()
        finally:
            os.dup2(saved, 2)
            os.close(saved)
        f.seek(0)
        return out, f.read()


def run(scale, ks, repeats, info):
    import torch
    from cugraph_b200 import pylibcugraph as plc
    from cugraph_b200.generators import rmat_edgelist
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    s2, d2 = torch.cat([src, dst]), torch.cat([dst, src])
    del src, dst
    h = plc.ResourceHandle()
    G = plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, store_transposed=False, renumber=True)
    E = int(s2.numel())
    del s2, d2
    V = 1 << scale
    for k in ks:
        n = V if k is None else k
        srcs = None if k is None else plc.select_random_vertices(h, G, 0, k)

        def call():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            plc.betweenness_centrality(h, G, srcs, None, True, False, False)
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        call()
        times = [call() * 1e3 for _ in range(repeats)]
        os.environ["CUGRAPH_B200_BC_TRACE"] = "1"
        h_tr = plc.ResourceHandle()  # the handle reads the knob when it is created
        os.environ.pop("CUGRAPH_B200_BC_TRACE")
        _, log = traced(lambda: plc.betweenness_centrality(h_tr, G, srcs, None, True, False, False))
        batches = [dict(zip(("sources", "levels", "bfs_ms", "sigma_ms", "backward_ms"),
                            (int(m[0]), int(m[1]), float(m[2]), float(m[3]), float(m[4]))))
                   for m in re.findall(r"sources (\d+) levels (\d+) entries \d+: bfs ([\d.]+) ms sigma ([\d.]+) ms "
                                       r"backward ([\d.]+) ms", log)]
        tot = {p: sum(b[p] for b in batches) for p in ("bfs_ms", "sigma_ms", "backward_ms")}
        best = min(times)
        out = {"workload": f"betweenness_rmat{scale}_ef16_sym_" + ("exact" if k is None else f"k{k}"), "vertices": V,
               "directed_edges": E, "sources": n, "call_ms": times, "batches": len(batches), "traced_split_ms": tot,
               "per_batch": batches[:4], "teps_best": n * E / (best / 1e3),
               "timing": "host clock around a synchronous call; split from CUDA events in a separate traced call"}
        out.update(info)
        print(json.dumps(out), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", type=int, nargs="*", default=[20, 24])
    ap.add_argument("--ks", type=int, nargs="*", default=[64, 256, 1024])
    ap.add_argument("--exact-scale", type=int, default=16)
    ap.add_argument("--repeats", type=int, default=2)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "betweenness_bench measures on the GPU"
    info = gpu_info()
    for sc in a.scales:
        run(sc, a.ks, a.repeats, info)
    if a.exact_scale:
        run(a.exact_scale, [None], a.repeats, info)
    return 0


if __name__ == "__main__":
    sys.exit(main())
