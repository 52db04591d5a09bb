"""Multi-source BFS against a loop of single-source BFS calls, on the graph of bench.py's traversal section.

RMAT-<scale> ef-16, symmetrised, renumbered, with bench.py's U[0,1) weights (ignored by BFS); the sources are bench.py's 64
timed BFS sources (non-isolated vertices, torch seed 1).  In one process:
  1. the distance rows of one cugraph_b200_multi_source_bfs call equal cugraph_bfs from each source alone;
  2. warm-up of both arms;
  3. one cugraph_b200_multi_source_bfs call over the sources against len(sources) cugraph_bfs calls
     (direction_optimizing=TRUE), the two arms alternated, --repeats times each;
  4. the same with one source, to show the fixed cost of a call.
Every timing is a host clock around synchronous C-ABI calls (each returns after a device synchronise), predecessors
computed in both arms, results freed outside the clock.  Prints one JSON line with the card's name, power limit and max SM
clock.  --trace: CUGRAPH_B200_BFS_TRACE=1, the per-level schedule and host time of every level on stderr.

    python scripts/multi_source_bfs_bench.py [--scale 24] [--sources 64] [--repeats 3] [--trace]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

INT_MAX = 2**31 - 1


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        return {"gpu_query_error": r.stderr.strip()[:200]}
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"card": name, "power_limit_w": float(power), "max_sm_clock_mhz": float(clock)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--sources", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--trace", action="store_true")
    a = ap.parse_args()
    if a.trace:
        os.environ["CUGRAPH_B200_BFS_TRACE"] = "1"
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200 import pylibcugraph as plc
    from cugraph_b200.generators import rmat_edgelist
    from cugraph_b200.pylibcugraph.utils import View, copy_to_torch
    L = _capi.lib()
    V = 1 << a.scale
    src, dst = rmat_edgelist(a.scale, 16 << a.scale, seed=0)
    s2, d2 = torch.cat([src, dst]), torch.cat([dst, src])
    del src, dst
    g = torch.Generator(device="cuda")
    g.manual_seed(2)
    w = torch.rand(s2.numel() // 2, device="cuda", generator=g)
    w2 = torch.cat([w, w])
    del w
    h = plc.ResourceHandle()
    G = plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, weight_array=w2,
                    store_transposed=False, renumber=True)
    deg = torch.bincount(s2.long(), minlength=V)
    e_sym = int(s2.numel())
    del s2, d2, w2
    cand = torch.nonzero(deg > 0).flatten()
    torch.manual_seed(1)
    sources = cand[torch.randperm(cand.numel(), device="cuda")[:a.sources + 1]].to(torch.int32)[1:].contiguous()

    def ms_call(s_t):
        """(seconds, result) of one cugraph_b200_multi_source_bfs call"""
        sv, res, err = View(s_t), C.c_void_p(), C.c_void_p()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        code = L.cugraph_b200_multi_source_bfs(h.ptr, G.ptr, sv.ptr, INT_MAX - 1, 1, C.byref(res), C.byref(err))
        dt = time.perf_counter() - t0
        sv.free()
        _capi.check(code, err, "cugraph_b200_multi_source_bfs")
        return dt, res

    def loop_call(s_t):
        """(seconds, results) of one cugraph_bfs call per source"""
        views = [View(s_t[i:i + 1]) for i in range(s_t.numel())]
        out = []
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for sv in views:
            res, err = C.c_void_p(), C.c_void_p()
            code = L.cugraph_bfs(h.ptr, G.ptr, sv.ptr, 1, INT_MAX - 1, 1, 0, C.byref(res), C.byref(err))
            _capi.check(code, err, "cugraph_bfs")
            out.append(res)
        dt = time.perf_counter() - t0
        for sv in views:
            sv.free()
        return dt, out

    def free(res):
        for r in (res if isinstance(res, list) else [res]):
            L.cugraph_paths_result_free(r)

    # 1. the rows against cugraph_bfs
    _, res = ms_call(sources)
    ms_verts = copy_to_torch(h, L.cugraph_paths_result_get_vertices(res))
    ms_dist = copy_to_torch(h, L.cugraph_paths_result_get_distances(res)).view(a.sources, ms_verts.numel())
    free(res)
    _, lres = loop_call(sources)
    rows_equal = True
    for k, r in enumerate(lres):
        verts = copy_to_torch(h, L.cugraph_paths_result_get_vertices(r))
        dist = copy_to_torch(h, L.cugraph_paths_result_get_distances(r))
        rows_equal = rows_equal and bool(torch.equal(verts, ms_verts)) and bool(torch.equal(dist, ms_dist[k]))
    free(lres)
    del ms_dist
    torch.cuda.empty_cache()
    # 2. warm-up, 3. the two arms alternated, 4. one source
    one = sources[:1].contiguous()
    for s_t in (sources, one):
        free(ms_call(s_t)[1])
        free(loop_call(s_t)[1])
    t_ms, t_loop, t_ms1, t_loop1 = [], [], [], []
    for _ in range(a.repeats):
        for s_t, t_a, t_b in ((sources, t_ms, t_loop), (one, t_ms1, t_loop1)):
            dt, res = ms_call(s_t)
            free(res)
            t_a.append(dt * 1e3)
            dt, res = loop_call(s_t)
            free(res)
            t_b.append(dt * 1e3)
    med = lambda x: sorted(x)[len(x) // 2]
    out = {"workload": f"multi_source_bfs_rmat{a.scale}_ef16_sym_{a.sources}_sources",
           "graph": f"RMAT-{a.scale} ef-16 symmetrised, {e_sym} directed edges", "sources": a.sources,
           "rows_equal_cugraph_bfs": rows_equal,
           "multi_source_ms": t_ms, f"cugraph_bfs_x{a.sources}_ms": t_loop,
           "one_source_multi_source_ms": t_ms1, "one_source_cugraph_bfs_ms": t_loop1,
           "median_speedup": med(t_loop) / med(t_ms),
           "timing": "host clock around synchronous C-ABI calls, arms alternated, predecessors computed in both"}
    out.update(gpu_info())
    print(json.dumps(out))
    return 0 if rows_equal else 1


if __name__ == "__main__":
    sys.exit(main())
