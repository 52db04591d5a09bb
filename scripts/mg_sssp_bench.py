"""Multi-GPU SSSP measurement (cugraph_b200.mg.MGGraph.sssp), one process per GPU under torchrun:

    torchrun --nproc-per-node N scripts/mg_sssp_bench.py --scale 24 --sources 8

Input: BASELINE's SSSP configuration, as bench.py builds it for one GPU: RMAT-`scale` ef-16 (seed 0) symmetrised, weights
U[0,1) from seed 2 (the same weight on both directions), sources = random non-isolated vertices from seed 1 (the first one is
the warm-up).  Every rank generates the edge list and keeps its share.
Parity first: MG = single GPU on RMAT-16 (distances bit-exact against cugraph_sssp on rank 0); a mismatch ends the run.
Timing: host clock around MGGraph.sssp, ending in a device synchronise, the max over ranks.  Graph500 TEPS per source =
undirected edges of the source's component / time.  Prints one JSON line on rank 0, with the card name and power limit read
in the same run."""
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


def _graph(scale, rank, world):
    from cugraph_b200.generators import rmat_edgelist
    V = 1 << scale
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    s2, d2 = torch.cat([src, dst]), torch.cat([dst, src])
    del src, dst
    g = torch.Generator(device="cuda")
    g.manual_seed(2)
    w = torch.rand(s2.numel() // 2, device="cuda", generator=g)
    w2 = torch.cat([w, w])
    del w
    deg = torch.bincount(s2.long(), minlength=V)
    cand = torch.nonzero(deg > 0).flatten()
    torch.manual_seed(1)
    sources = cand[torch.randperm(cand.numel(), device="cuda")].tolist()
    E = s2.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    return s2[lo:hi].clone(), d2[lo:hi].clone(), w2[lo:hi].clone(), deg, sources, (s2, d2, w2) if rank == 0 else None


def _gather_dist(verts, d, V):
    """distances of all vertices by id on rank 0 (ids that are not vertices of the graph: FLT_MAX)"""
    parts = [None] * dist.get_world_size()
    dist.all_gather_object(parts, (verts.cpu(), d.cpu()))
    out = torch.full((V,), torch.finfo(d.dtype).max, dtype=d.dtype)
    for v, x in parts:
        out[v.long()] = x
    return out


def parity(groups, scale=16):
    from cugraph_b200 import mg
    from cugraph_b200 import pylibcugraph as plc
    rank, world = dist.get_rank(), dist.get_world_size()
    s, d, w, _, sources, full = _graph(scale, rank, world)
    G = mg.MGGraph(s, d, w, groups)
    src = sources[0]
    verts, dd, _ = G.sssp(src, compute_predecessors=False)
    got = _gather_dist(verts, dd, 1 << scale)
    del G
    if rank != 0:
        return None
    s2, d2, w2 = full
    h = plc.ResourceHandle()
    g1 = plc.SGGraph(h, plc.GraphProperties(is_symmetric=True, is_multigraph=True), s2, d2, weight_array=w2,
                     store_transposed=False, renumber=True)
    v1, d1, _ = plc.sssp(h, g1, src, float("inf"), False, False)
    ref = torch.full((1 << scale,), torch.finfo(torch.float32).max, dtype=torch.float32)
    ref[v1.cpu().long()] = d1.cpu()
    return {"ok": bool(torch.equal(got, ref)), "scale": scale, "source": src,
            "reached": int((ref < torch.finfo(torch.float32).max).sum())}


def _card(local):
    name = torch.cuda.get_device_name(local)
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(local)],
                           capture_output=True, text=True, timeout=30)
        power = float(r.stdout.strip().splitlines()[0])
    except Exception:  # noqa: BLE001
        power = None
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--sources", type=int, default=8)
    args = ap.parse_args()
    from cugraph_b200 import mg
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29531")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    groups = mg.make_groups()
    par = parity(groups)
    ok = torch.tensor([1 if (rank != 0 or par["ok"]) else 0], dtype=torch.int32, device="cuda")
    dist.broadcast(ok, src=0)
    if int(ok.item()) == 0:
        raise SystemExit(f"multi-GPU SSSP does not match the single-GPU result: {par}")
    s, d, w, deg, sources, _ = _graph(args.scale, rank, world)
    G = mg.MGGraph(s, d, w, groups)
    del s, d, w
    torch.cuda.empty_cache()
    ms, teps, rounds, windows = [], [], [], []
    for i in range(args.sources + 1):           # source 0 is the warm-up
        dist.barrier()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        verts, dd, _ = G.sssp(sources[i], compute_predecessors=False)
        torch.cuda.synchronize()
        dt = torch.tensor([time.perf_counter() - t0], dtype=torch.float64, device="cuda")
        dist.all_reduce(dt, op=dist.ReduceOp.MAX)
        ne = deg[verts.long()][dd < torch.finfo(dd.dtype).max].sum().reshape(1)
        dist.all_reduce(ne)
        if i == 0:
            continue
        t = float(dt.item())
        ms.append(t * 1e3)
        teps.append(int(ne.item()) // 2 / t)
        rounds.append(G.last_sssp_stats["rounds"])
        windows.append(G.last_sssp_stats["windows"])
    name, power = _card(local)
    if rank == 0:
        out = {"metric": f"MG SSSP RMAT-{args.scale} ef-16 symmetrised, Graph500 TEPS", "n_gpus": world,
               "grid": f"{groups.R}x{groups.C}", "sources": args.sources, "ms_per_source": sum(ms) / len(ms),
               "ms_min_max": [min(ms), max(ms)], "rounds_mean": sum(rounds) / len(rounds),
               "windows_mean": sum(windows) / len(windows),
               "gteps_harmonic": len(teps) / sum(1.0 / x for x in teps) / 1e9, "gteps_mean": sum(teps) / len(teps) / 1e9,
               "parity": par, "card": name, "power_limit_w": power,
               "timing": "host clock around MGGraph.sssp ending in a device synchronise, max over ranks"}
        print(json.dumps(out), flush=True)
    del G
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
