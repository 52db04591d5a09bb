"""Multi-GPU BFS from a set of sources and multi-GPU extract_paths measurement (cugraph_b200.mg.MGGraph.bfs /
.extract_paths), one process per GPU under torchrun:

    torchrun --nproc-per-node N scripts/mg_paths_bench.py --scale 24 --calls 5

Input: BASELINE's BFS configuration, as bench.py builds it for one GPU: RMAT-`scale` ef-16 (seed 0) symmetrised, unweighted.
Every rank generates the edge list and keeps its share.
Cases: MG BFS from 1 and from 64 sources (random vertices with edges, seed 1; the 64 dealt round-robin to the ranks) in
three schedules: top-down on every level (bfs_<k>_sources, MGGraph.bfs's default), direction-optimising
(bfs_<k>_sources_optimizing) and every level bottom-up (bfs_<k>_sources_all_bottom_up: direction_optimizing=True on a
second MGGraph built under CUGRAPH_B200_BFS_ALPHA = CUGRAPH_B200_BFS_BETA = 1e30), each with its last_bfs_stats; then
extract_paths of 2^16 random vertices (dealt the same way) and of every vertex (each rank its own vertices) on the
64-source top-down result.  Single GPU (world size 1 only: the whole graph on one GPU): cugraph_bfs from the same sources and
cugraph_extract_paths of the same destinations, the same way.
Parity first: on RMAT-16 from 64 sources, the MG distances of the top-down and the direction-optimising schedule must equal
single-GPU cugraph_bfs's and the MG max_path_length cugraph_extract_paths' on rank 0; a mismatch ends the run.
Timing: one warm-up call, then `calls` timed calls, each with a host clock that ends in a device synchronise, the max over
ranks.  Prints one JSON line on rank 0 (ms per call, position rounds of each extract_paths case), with the card name and
power limit read in the same run.  --backend gloo runs the same steps over gloo (a functional check of the script)."""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

INT32_MAX = 2**31 - 1


def _graph(scale, rank, world):
    from cugraph_b200.generators import rmat_edgelist
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    s2, d2 = torch.cat([src, dst]), torch.cat([dst, src])
    del src, dst
    E = s2.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    return s2[lo:hi].clone(), d2[lo:hi].clone(), (s2, d2) if rank == 0 else None


def _picks(scale, k, seed):
    """k distinct random vertex ids with at least one edge, the same on every rank"""
    from cugraph_b200.generators import rmat_edgelist
    src, _ = rmat_edgelist(scale, 16 << scale, seed=0)
    ids = torch.unique(src.cpu())
    g = torch.Generator().manual_seed(seed)
    return ids[torch.randperm(ids.numel(), generator=g)[:k]].to(torch.int32)


def _deal(ids, rank, world):
    return ids[rank::world].contiguous().to("cuda")


def _single_gpu(s2, d2):
    from cugraph_b200 import pylibcugraph as plc
    h = plc.ResourceHandle()
    g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, store_transposed=False,
                    renumber=True)
    return h, g


class _SG:
    """single-GPU cugraph_bfs + cugraph_extract_paths through the C ABI (the paths result feeds extract_paths)"""

    def __init__(self, s2, d2):
        from cugraph_b200 import _capi
        self.h, self.g = _single_gpu(s2, d2)
        self.L, self.capi = _capi.lib(), _capi
        self.res = None

    def bfs(self, sources):
        from cugraph_b200.pylibcugraph.utils import View
        self.free()
        sv, res, err = View(sources), C.c_void_p(), C.c_void_p()
        self.h.order_after_caller()
        code = self.L.cugraph_bfs(self.h.ptr, self.g.ptr, sv.ptr, 0, INT32_MAX - 1, 1, 0, C.byref(res), C.byref(err))
        sv.free()
        self.capi.check(code, err, "cugraph_bfs")
        self.res = res

    def distances(self):
        from cugraph_b200.pylibcugraph.utils import copy_to_torch
        v = copy_to_torch(self.h, self.L.cugraph_paths_result_get_vertices(self.res)).long().cpu()
        d = copy_to_torch(self.h, self.L.cugraph_paths_result_get_distances(self.res)).long().cpu()
        out = torch.full((int(v.max()) + 1,), -1, dtype=torch.int64)
        out[v] = d
        return out

    def extract_paths(self, dests):
        from cugraph_b200.pylibcugraph.utils import View
        dv, out, err = View(dests), C.c_void_p(), C.c_void_p()
        code = self.L.cugraph_extract_paths(self.h.ptr, self.g.ptr, dv.ptr, self.res, dv.ptr, C.byref(out), C.byref(err))
        dv.free()
        self.capi.check(code, err, "cugraph_extract_paths")
        n = int(self.L.cugraph_extract_paths_result_get_max_path_length(out))
        self.L.cugraph_extract_paths_result_free(out)
        return n

    def free(self):
        if self.res is not None:
            self.L.cugraph_paths_result_free(self.res)
            self.res = None


def parity(groups, scale=16):
    from cugraph_b200 import mg
    rank, world = dist.get_rank(), dist.get_world_size()
    s, d, full = _graph(scale, rank, world)
    srcs = _picks(scale, 64, 1)
    dests = _picks(scale, 4096, 2)
    G = mg.MGGraph(s, d, None, groups)
    v, dd, pred = G.bfs(_deal(srcs, rank, world))
    _, length = G.extract_paths(dd, pred, _deal(dests, rank, world))
    _, dd_opt, _ = G.bfs(_deal(srcs, rank, world), direction_optimizing=True)
    parts = [None] * world
    dist.all_gather_object(parts, (v.cpu(), dd.cpu(), dd_opt.cpu()))
    del G
    if rank != 0:
        return None
    sg = _SG(*full)
    sg.bfs(srcs.to("cuda"))
    ref = sg.distances()
    sg_len = sg.extract_paths(dests.to("cuda"))
    sg.free()
    same = all(torch.equal(ref[pv.long()], pd.long()) and torch.equal(pd, po) for pv, pd, po in parts)
    return {"ok": bool(same and sg_len == length), "scale": scale, "max_path_length": length}


def _card(local):
    try:
        name = torch.cuda.get_device_name(local)
    except Exception:  # noqa: BLE001
        name = None
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(local)],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        power = None
    return name, power


def _timed(fn):
    dist.barrier()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device="cuda")
    dist.all_reduce(dt, op=dist.ReduceOp.MAX)
    return float(dt.item()) * 1e3, out


def _series(fn, calls):
    ms, out = [], None
    for i in range(calls + 1):            # call 0 is the warm-up
        t, out = _timed(fn)
        if i:
            ms.append(t)
    return dict(ms_per_call=sum(ms) / len(ms), ms_min_max=[min(ms), max(ms)]), out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--parity-scale", type=int, default=16)
    ap.add_argument("--backend", default="nccl")
    args = ap.parse_args(argv)
    from cugraph_b200 import mg
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    torch.cuda.set_device(local)
    if args.backend == "nccl":
        dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    else:
        dist.init_process_group(args.backend, rank=rank, world_size=world)
    groups = mg.make_groups()
    par = parity(groups, args.parity_scale)
    ok = torch.tensor([1 if (rank != 0 or par["ok"]) else 0], dtype=torch.int32, device="cuda")
    dist.broadcast(ok, src=0)
    if int(ok.item()) == 0:
        raise SystemExit(f"multi-GPU BFS / extract_paths do not match single GPU: {par}")
    srcs = {1: _picks(args.scale, 1, 1), 64: _picks(args.scale, 64, 1)}
    dests16 = _picks(args.scale, 1 << 16, 2)
    s, d, full = _graph(args.scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    del s, d
    torch.cuda.empty_cache()
    mg_res = {}
    for k, src in srcs.items():
        mine = _deal(src, rank, world)
        mg_res[f"bfs_{k}_sources_optimizing"], _ = _series(lambda: G.bfs(mine, direction_optimizing=True), args.calls)
        mg_res[f"bfs_{k}_sources_optimizing"].update(G.last_bfs_stats)
        mg_res[f"bfs_{k}_sources"], last = _series(lambda: G.bfs(mine), args.calls)
        mg_res[f"bfs_{k}_sources"].update(G.last_bfs_stats)
    _, dd, pred = last
    for name, dests in (("paths_2^16", _deal(dests16, rank, world)), ("paths_all", G.part.vertices)):
        mg_res[name], (_, length) = _series(lambda: G.extract_paths(dd, pred, dests), args.calls)
        mg_res[name].update(rounds=G.last_paths_stats["rounds"], max_path_length=length)
    del G, dd, pred, last
    torch.cuda.empty_cache()
    # every level bottom-up: the knobs are read when the graph's handle is made
    knobs = {k: os.environ.get(k) for k in ("CUGRAPH_B200_BFS_ALPHA", "CUGRAPH_B200_BFS_BETA")}
    os.environ.update({k: "1e30" for k in knobs})
    s, d, _ = _graph(args.scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    del s, d
    for k, v in knobs.items():
        if v is None:
            os.environ.pop(k)
        else:
            os.environ[k] = v
    for k, src in srcs.items():
        mine = _deal(src, rank, world)
        mg_res[f"bfs_{k}_sources_all_bottom_up"], _ = _series(lambda: G.bfs(mine, direction_optimizing=True), args.calls)
        mg_res[f"bfs_{k}_sources_all_bottom_up"].update(G.last_bfs_stats)
    del G
    torch.cuda.empty_cache()
    sg_res = None
    if world == 1:
        sg_res = {}
        sg = _SG(*full)
        for k, src in srcs.items():
            sg_res[f"bfs_{k}_sources"], _ = _series(lambda: sg.bfs(src.to("cuda")), args.calls)
        all_ids = full[0].unique() if full[0].numel() else full[0]
        for name, dests in (("paths_2^16", dests16.to("cuda")), ("paths_all", all_ids)):
            sg_res[name], length = _series(lambda: sg.extract_paths(dests), args.calls)
            sg_res[name].update(max_path_length=length)
        sg.free()
    del full
    name, power = _card(local)
    if rank == 0:
        out = {"metric": f"MG BFS / extract_paths RMAT-{args.scale} ef-16 symmetrised, ms per call", "n_gpus": world,
               "grid": f"{groups.R}x{groups.C}", "calls": args.calls, "mg": mg_res, "single_gpu": sg_res, "parity": par,
               "card": name, "power_limit_w": power,
               "timing": "host clock around the call ending in a device synchronise, max over ranks"}
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
