"""Graph500 BFS and SSSP on the 2D partition (cugraph_b200.mg.MGGraph), one process per GPU under torchrun:

    torchrun --nproc-per-node N scripts/graph500.py --scale 24 [--roots 64] [--no-direction-optimizing] [--single-gpu]

World size 1 is the 1x1 grid.
  Kernel 1 (construction): every rank generates its slice of RMAT-`scale`, edge factor 16, seed 0
    (mg.rmat_edgelist_share: the same global edge stream whatever the world size), float32 weights U[0,1) drawn at the same
    global indices (generators.uniform_values, seed 2), and adds the reversed copy of every tuple with the same weight; the
    MGGraph built from these (no drop options) is bench.py's traversal graph, built in slices.  The slices are freed after
    construction.  Time: host clock from the slices to the graph, barrier and device synchronise on both sides, max over
    ranks.
  Roots: `--roots` distinct vertices of degree >= 1, drawn in order from a counter-based integer stream (seed 3) and checked
    at their owners through MGGraph.degrees().  Graph500 also excludes vertices whose only edges are self-loops; such a
    vertex can be picked here.
  Kernel 2: per root, MGGraph.bfs(root, direction_optimizing=...) timed like kernel 1, then MGGraph.validate_bfs.
  Kernel 3: per root, MGGraph.sssp(root) timed the same way, then MGGraph.validate_sssp.
  TEPS per root = edges_from_reached / 2 over the time: the input tuples of the root's component, self-loops and
    duplicates included (Graph500's count, bench.py's sum of degrees / 2).
  --single-gpu (world size 1 only): after the multi-GPU kernels, also the SGGraph of bench.py's traversal from the same
    tuples generated again (so that the multi-GPU construction's temporaries are gone by then); cugraph_bfs /
    cugraph_sssp through the C ABI from the same roots, timed around the call, every result validated on the 1x1 MGGraph.
Validation runs outside the timed calls.  Rank 0 prints one JSON line; a root that fails validation makes the script exit
non-zero after it."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import math
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EDGE_FACTOR = 16
WEIGHT_SEED, ROOT_SEED = 2, 3


def _sync_max(value, D):
    """the max of a host float over the ranks (one all-reduce)"""
    t = torch.tensor([float(value)], dtype=torch.float64, device="cuda")
    D.all_reduce(t, op=D.ReduceOp.MAX)
    return float(t.item())


def _barrier(D):
    """every rank gets here before any goes on (an all-reduce: also the in-process stand-in has no barrier)"""
    D.all_reduce(torch.zeros(1, dtype=torch.float64, device="cuda"))
    torch.cuda.synchronize()


def _timed(fn, D):
    """fn() with a barrier and a device synchronise on both sides: (result, its wall seconds as the max over ranks)"""
    _barrier(D)
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, _sync_max(time.perf_counter() - t0, D)


def _roots(G, n_roots, V, D):
    """n_roots distinct vertices of degree >= 1, the same on every rank: candidates from the counter-based int32 stream of
    ROOT_SEED over [0, V), in order, kept when their owner finds them with an out-degree >= 1"""
    from cugraph_b200.generators import uniform_values
    verts, _, out_deg = G.degrees()
    order = torch.argsort(verts.to(torch.int64))
    sv, sd = verts.to(torch.int64)[order], out_deg.to(torch.int64)[order]
    picked, first, batch = [], 0, max(4 * n_roots, 64)
    while len(picked) < n_roots and first < 64 * V:
        cand = uniform_values(batch, ROOT_SEED, 0, V, torch.int32, first=first).to(torch.int64)
        first += batch
        ok = torch.zeros(batch, dtype=torch.int64, device=cand.device)
        if sv.numel():
            pos = torch.searchsorted(sv, cand).clamp(max=sv.numel() - 1)
            ok = ((sv[pos] == cand) & (sd[pos] > 0)).to(torch.int64)
        D.all_reduce(ok, op=D.ReduceOp.MAX)
        for c, k in zip(cand.tolist(), ok.tolist()):
            if k and c not in picked and len(picked) < n_roots:
                picked.append(c)
    return picked


def _stats(times, edges):
    """time quartiles, mean and stddev; TEPS harmonic mean and Graph500's harmonic stddev"""
    n = len(times)
    if n == 0:
        return {}
    ts = sorted(times)

    def q(f):   # linear interpolation between order statistics
        x = f * (n - 1)
        lo = int(math.floor(x))
        hi = min(lo + 1, n - 1)
        return ts[lo] + (ts[hi] - ts[lo]) * (x - lo)

    mean = sum(ts) / n
    sd = math.sqrt(sum((t - mean) ** 2 for t in ts) / (n - 1)) if n > 1 else 0.0
    teps = [e / 2 / t for e, t in zip(edges, times)]
    out = {"time_s": {"min": ts[0], "q1": q(0.25), "median": q(0.5), "q3": q(0.75), "max": ts[-1], "mean": mean,
                      "stddev": sd}}
    if all(x > 0 for x in teps):
        hm = n / sum(1.0 / x for x in teps)
        hsd = (math.sqrt(sum((1.0 / x - 1.0 / hm) ** 2 for x in teps) / (n - 1)) * hm * hm / math.sqrt(n)) if n > 1 else 0.0
        out["teps"] = {"harmonic_mean": hm, "harmonic_stddev": hsd, "min": min(teps), "max": max(teps)}
    return out


def _kernel(run_one, check_one, roots, D, keep, fetch=None):
    """per root: the timed call, then (fetch: reading its result back) its validation, timed apart; returns (summary,
    per-root kept results)"""
    times, edges, check_s, n_ok, failed, kept = [], [], [], 0, [], []
    for root in roots:
        res, dt = _timed(lambda: run_one(root), D)
        if fetch is not None:
            res = fetch(res)
        t0 = time.perf_counter()
        cert = check_one(root, res)
        check_s.append(_sync_max(time.perf_counter() - t0, D))
        times.append(dt)
        edges.append(cert["edges_from_reached"])
        if cert["ok"]:
            n_ok += 1
        else:
            failed.append({"root": root, **{k: v for k, v in cert.items() if v and k != "edges_from_reached"}})
        if keep:
            kept.append((res[0].cpu(), res[1].cpu(), cert["edges_from_reached"]))
    out = {"roots": len(roots), "validated": n_ok, **_stats(times, edges),
           "validation_s_per_root": sum(check_s) / len(check_s) if check_s else None}
    if failed:
        out["failed"] = failed[:8]
    return out, kept


def _single_gpu_calls(scale, s2, d2, w2, direction_optimizing):
    """bench.py's traversal SGGraph over the same arrays and the C-ABI calls on it: (bfs(root), sssp(root)) -> (vertices,
    distances, predecessors)"""
    from cugraph_b200 import _capi
    from cugraph_b200 import pylibcugraph as plc
    from cugraph_b200.pylibcugraph.utils import View, copy_to_torch
    L = _capi.lib()
    h = plc.ResourceHandle()
    SG = plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, weight_array=w2,
                     store_transposed=False, renumber=True)
    imax = 2**31 - 1

    def read(res):
        out = tuple(copy_to_torch(h, getattr(L, f"cugraph_paths_result_get_{k}")(res))
                    for k in ("vertices", "distances", "predecessors"))
        L.cugraph_paths_result_free(res)
        return out

    def bfs(root):
        res, err = C.c_void_p(), C.c_void_p()
        sv = View(torch.tensor([root], dtype=torch.int32, device="cuda"))
        code = L.cugraph_bfs(h.ptr, SG.ptr, sv.ptr, 1 if direction_optimizing else 0, imax - 1, 1, 0, C.byref(res),
                             C.byref(err))
        sv.free()
        _capi.check(code, err, "cugraph_bfs")
        return res

    def sssp(root):
        res, err = C.c_void_p(), C.c_void_p()
        code = L.cugraph_sssp(h.ptr, SG.ptr, int(root), float("inf"), 1, 0, C.byref(res), C.byref(err))
        _capi.check(code, err, "cugraph_sssp")
        return res

    return SG, h, bfs, sssp, read


def run(groups, scale, n_roots=64, direction_optimizing=True, single_gpu=False, keep_results=False):
    """The harness on the grid of `groups` (mg.make_groups()): returns the result dict, the same on every rank.  With
    keep_results the dict also holds, under "results", this rank's (vertices, distances, edges_from_reached) per root and
    kernel, on the host."""
    from cugraph_b200 import mg
    from cugraph_b200.generators import uniform_values
    D = mg.dist
    E = EDGE_FACTOR << scale
    if single_gpu and groups.world != 1:
        raise ValueError("--single-gpu needs world size 1")
    def tuples():
        """this rank's slice of the input tuples and their weights, drawn at the same global indices"""
        src, dst, first = mg.rmat_edgelist_share(scale, E, seed=0, groups=groups)
        return src, dst, uniform_values(src.numel(), WEIGHT_SEED, 0.0, 1.0, torch.float32, device=src.device, first=first)

    src, dst, w = tuples()
    G, t_build = _timed(lambda: mg.MGGraph(torch.cat([src, dst]), torch.cat([dst, src]), torch.cat([w, w]), groups), D)
    del src, dst, w
    torch.cuda.empty_cache()       # the shuffle's temporaries go back to the driver
    roots = _roots(G, n_roots, 1 << scale, D)
    out = {"scale": scale, "edge_factor": EDGE_FACTOR, "grid": f"{groups.R}x{groups.C}", "n_gpus": groups.world,
           "roots": len(roots), "direction_optimizing": bool(direction_optimizing),
           "root_rule": "distinct vertices of degree >= 1 (a vertex whose only edges are self-loops can be picked; "
                        "Graph500 excludes those)",
           "construction_s": t_build}
    kept = {}
    out["bfs"], kept["bfs"] = _kernel(
        lambda r: G.bfs(r, direction_optimizing=direction_optimizing),
        lambda r, res: G.validate_bfs(res[0], res[1], res[2], r), roots, D, keep_results)
    out["sssp"], kept["sssp"] = _kernel(
        lambda r: G.sssp(r), lambda r, res: G.validate_sssp(res[0], res[1], res[2], r), roots, D, keep_results)
    if single_gpu:
        # built after the multi-GPU kernels, from the same tuples generated again: the construction's temporaries are gone,
        # and the two graphs share the device only while the single-GPU results are timed and validated
        src, dst, w = tuples()
        SG, h, bfs, sssp, read = _single_gpu_calls(scale, torch.cat([src, dst]), torch.cat([dst, src]), torch.cat([w, w]),
                                                   direction_optimizing)
        del src, dst, w
        torch.cuda.empty_cache()
        out["single_gpu"] = {}
        for name, call, check in (("bfs", bfs, G.validate_bfs), ("sssp", sssp, G.validate_sssp)):
            out["single_gpu"][name], kept["single_gpu_" + name] = _kernel(
                call, lambda r, res, check=check: check(*res, r), roots, D, keep_results, fetch=read)
        del SG, bfs, sssp, read
    out["timing"] = ("host clock around each call with a barrier and a device synchronise on both sides, max over ranks; "
                     "validation outside the timed calls")
    out["ok"] = all(k["validated"] == k["roots"] for k in [out["bfs"], out["sssp"]] + list(out.get("single_gpu", {}).values()))
    if keep_results:
        out["results"] = kept
    del G
    return out


def _card(local):
    """device name, power limit (W) and max SM clock (MHz) of the local GPU, read in this run"""
    name = torch.cuda.get_device_name(local)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i",
                            str(local)], capture_output=True, text=True, timeout=30)
        power, clock = (float(x) for x in r.stdout.strip().splitlines()[0].split(","))
    except Exception:  # noqa: BLE001
        power = clock = None
    return name, power, clock


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--roots", type=int, default=64)
    ap.add_argument("--direction-optimizing", dest="direction_optimizing", action="store_true", default=True)
    ap.add_argument("--no-direction-optimizing", dest="direction_optimizing", action="store_false")
    ap.add_argument("--single-gpu", action="store_true")
    args = ap.parse_args()
    import torch.distributed as dist
    from cugraph_b200 import mg
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    if args.single_gpu and world != 1:
        raise SystemExit("--single-gpu needs world size 1")
    out = run(mg.make_groups(), args.scale, args.roots, args.direction_optimizing, args.single_gpu)
    out["card"], out["power_limit_w"], out["max_sm_clock_mhz"] = _card(local)
    if rank == 0:
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()
    if not out["ok"]:
        raise SystemExit(1)


if __name__ == "__main__":
    main()
