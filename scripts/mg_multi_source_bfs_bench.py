"""Multi-GPU multi-source BFS (cugraph_b200.mg.MGGraph.multi_source_bfs) against one MGGraph.bfs call per source, one
process per GPU under torchrun:

    torchrun --nproc-per-node N scripts/mg_multi_source_bfs_bench.py --scale 24 --repeats 3

Input: bench.py's BFS configuration: RMAT-`scale` ef-16 (seed 0) symmetrised, unweighted, and its 64 BFS sources (vertices
with edges, torch seed 1).  Every rank generates the edge list and keeps its share.
1. Parity on symmetrised RMAT-16: every row of one multi_source_bfs call (top-down and direction-optimising) equals
   MGGraph.bfs from that source alone (distances and predecessors) and, on a world of one, the distance row of single-GPU
   cugraph_b200_multi_source_bfs.  A mismatch ends the run.
2. At --scale, the arms, alternated, one warm-up call each, then --repeats timed calls: one multi_source_bfs call top-down,
   the same with direction_optimizing=True, the same top-down without predecessors, len(sources) MGGraph.bfs calls, and on a
   world of one a single-GPU cugraph_b200_multi_source_bfs call.  Each time is a host clock that ends in a device
   synchronise, the max over ranks.
Prints one JSON line on rank 0: ms per call (min-max and all), the levels per direction, the card name and power limit
read in the same run.  --backend gloo runs the same steps over gloo on the CPU (a functional check of the script)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True)
    if r.returncode != 0:
        return {"gpu_query_error": r.stderr.strip()[:200]}
    name, power, clock = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
    return {"card": name, "power_limit_w": float(power), "max_sm_clock_mhz": float(clock)}


def edges(scale):
    """bench.py's symmetrised RMAT edge list and its BFS sources (the same on every rank)"""
    from cugraph_b200.generators import rmat_edgelist
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    s2, d2 = torch.cat([src, dst]), torch.cat([dst, src])
    del src, dst
    deg = torch.bincount(s2.long(), minlength=1 << scale)
    cand = torch.nonzero(deg > 0).flatten()
    torch.manual_seed(1)
    sources = cand[torch.randperm(cand.numel(), device=cand.device)[:65]].to(torch.int32)[1:].contiguous()
    return s2, d2, sources


def build(scale, rank, world):
    from cugraph_b200 import mg
    s2, d2, sources = edges(scale)
    E = s2.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    g = mg.MGGraph(s2[lo:hi].clone(), d2[lo:hi].clone())
    whole = (s2, d2) if world == 1 else None
    if whole is None:
        del s2, d2
    return g, sources, whole


def single_gpu(s2, d2):
    from cugraph_b200 import pylibcugraph as plc
    h = plc.ResourceHandle()
    return h, plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, store_transposed=False,
                          renumber=True)


def timed(fn):
    torch.cuda.synchronize()
    dist.barrier()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    t = torch.tensor([(time.perf_counter() - t0) * 1e3], dtype=torch.float64, device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item()), out


def parity(rank, world):
    from cugraph_b200.traversal import multi_source_bfs as sg_ms_bfs
    g, sources, whole = build(16, rank, world)
    ok = True
    for do in (False, True):
        v, d, p = g.multi_source_bfs(sources.cuda(), direction_optimizing=do)
        for k in range(sources.numel()):
            _, d1, p1 = g.bfs(int(sources[k]))
            ok = ok and bool(torch.equal(d[k], d1) and torch.equal(p[k], p1))
        if whole is not None:
            h, G = single_gpu(*whole)
            sd, _, sv = sg_ms_bfs(h, G, sources.cuda(), 0, False)
            pos = torch.searchsorted(sv.long().sort().values, v.long())
            order = sv.long().argsort()
            ok = ok and bool(torch.equal(sd[:, order[pos]], d))
    flag = torch.tensor([0 if ok else 1], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MAX)
    return int(flag.item()) == 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--backend", default="nccl")
    a = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    if a.backend == "nccl":
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    else:
        dist.init_process_group("gloo")
    out = {"workload": f"mg_multi_source_bfs_rmat{a.scale}_ef16_sym_64_sources", "world": world}
    out["parity_rmat16"] = parity(rank, world)
    if not out["parity_rmat16"]:
        if rank == 0:
            print(json.dumps(out))
        dist.destroy_process_group()
        return 1
    torch.cuda.empty_cache()
    g, sources, whole = build(a.scale, rank, world)
    src = sources.cuda()
    levels = {}

    def ms(do, pred=True):
        def run():
            r = g.multi_source_bfs(src, compute_predecessors=pred, direction_optimizing=do)
            levels["optimizing" if do else "top_down"] = dict(g.last_ms_bfs_stats)
            return r
        return run

    def loop():
        for k in range(src.numel()):
            g.bfs(int(sources[k]))

    arms = {"multi_source_top_down": ms(False), "multi_source_optimizing": ms(True),
            "multi_source_top_down_no_predecessors": ms(False, False), "mg_bfs_x64": loop}
    if whole is not None:
        from cugraph_b200.traversal import multi_source_bfs as sg_ms_bfs
        h, G = single_gpu(*whole)
        arms["single_gpu_multi_source"] = lambda: sg_ms_bfs(h, G, src, 0, True)
    times = {k: [] for k in arms}
    for name, fn in arms.items():   # warm-up
        timed(fn)
        torch.cuda.empty_cache()
    for _ in range(a.repeats):
        for name, fn in arms.items():
            t, _ = timed(fn)
            times[name].append(t)
            torch.cuda.empty_cache()
    for name, ts in times.items():
        out[f"{name}_ms"] = ts
        out[f"{name}_ms_min_max"] = [min(ts), max(ts)]
    out["levels"] = levels
    out["timing"] = "host clock ending in a device synchronise, max over ranks, arms alternated, one warm-up call each"
    out.update(gpu_info() if a.backend == "nccl" else {})
    if rank == 0:
        print(json.dumps(out))
    dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
