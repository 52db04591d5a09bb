"""Multi-GPU strongly connected components measurement (cugraph_b200.mg.MGGraph.strongly_connected_components), one process
per GPU under torchrun:

    torchrun --nproc-per-node N scripts/mg_scc_bench.py --scale 24 --calls 5 [--per-phase]

Input: scripts/scc_bench.py's graph: directed RMAT-`scale` from the library's device generator (seed 0), edge factor 16,
as generated (multi-edges and self-loops kept), unweighted.  Every rank generates the edge list and keeps its share.
Parity first: on RMAT-16, the MG components must be the same partition as single-GPU cugraph_strongly_connected_components
on rank 0; a mismatch ends the run.
Timing: one warm-up call, then `calls` timed calls, each with a host clock that ends in a device synchronise, the max over
ranks.  Single-GPU SCC on the same graph, the same way, on rank 0 (world size 1 only: the whole graph on one GPU).
--per-phase adds one extra call that synchronises around every phase (trim, forward-backward, colouring, labels) and
records its time, next to the call's rounds (last_scc_stats).
Prints one JSON line on rank 0, with the card name and power limit read in the same run."""
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
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    E = src.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    return src[lo:hi].clone(), dst[lo:hi].clone(), (src, dst) if rank == 0 else None


def _gather_labels(verts, labels, V):
    """labels of all vertices by id on rank 0 (ids that are not vertices of the graph: their own id)"""
    parts = [None] * dist.get_world_size()
    dist.all_gather_object(parts, (verts.cpu(), labels.cpu()))
    out = torch.arange(V, dtype=torch.int64)
    for v, x in parts:
        out[v.long()] = x.long()
    return out


def _same_partition(a, b):
    pairs = torch.unique(torch.stack([a, b]), dim=1)
    return pairs.shape[1] == torch.unique(a).numel() == torch.unique(b).numel()


def _single_gpu(src, dst, V):
    from cugraph_b200 import pylibcugraph as plc
    h = plc.ResourceHandle()
    g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=False, is_multigraph=True), src, dst, store_transposed=False,
                    renumber=True, vertices_array=torch.arange(V, dtype=torch.int32, device="cuda"))
    return h, g


def parity(groups, scale=16):
    from cugraph_b200 import mg
    from cugraph_b200 import pylibcugraph as plc
    rank, world = dist.get_rank(), dist.get_world_size()
    V = 1 << scale
    s, d, full = _graph(scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    verts, labels = G.strongly_connected_components()
    got = _gather_labels(verts, labels, V)
    del G
    if rank != 0:
        return None
    h, g1 = _single_gpu(*full, V)
    v1, l1 = plc.strongly_connected_components(h, g1, None, None, None, None, False)
    ref = torch.arange(V, dtype=torch.int64)
    ref[v1.cpu().long()] = l1.cpu().long()
    return {"ok": bool(_same_partition(got, ref)), "scale": scale, "components": int(torch.unique(ref).numel())}


def _card(local):
    name = torch.cuda.get_device_name(local)
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


def per_phase(G):
    """one call with every phase of _SccRun timed on its own (synchronised, max over ranks), with the call's rounds"""
    from cugraph_b200 import mg
    names = ("trim", "forward_backward", "colouring", "labels")
    saved = {n: getattr(mg._SccRun, n) for n in names}
    ms = {}

    def timing(name, fn):
        def wrapper(run):
            t, out = _timed(lambda: fn(run))
            ms[name] = round(t, 3)
            return out
        return wrapper

    for n in names:
        setattr(mg._SccRun, n, timing(n, saved[n]))
    try:
        G.strongly_connected_components()
    finally:
        for n in names:
            setattr(mg._SccRun, n, saved[n])
    return {"phase_ms": ms, "rounds": G.last_scc_stats}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--per-phase", action="store_true")
    args = ap.parse_args()
    from cugraph_b200 import mg
    from cugraph_b200 import pylibcugraph as plc
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29533")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    groups = mg.make_groups()
    par = parity(groups)
    ok = torch.tensor([1 if (rank != 0 or par["ok"]) else 0], dtype=torch.int32, device="cuda")
    dist.broadcast(ok, src=0)
    if int(ok.item()) == 0:
        raise SystemExit(f"multi-GPU SCC does not give the single-GPU components: {par}")
    V = 1 << args.scale
    s, d, full = _graph(args.scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    del s, d
    torch.cuda.empty_cache()
    ms = []
    for i in range(args.calls + 1):            # call 0 is the warm-up
        t, _ = _timed(G.strongly_connected_components)
        if i:
            ms.append(t)
    rounds = G.last_scc_stats
    phases = per_phase(G) if args.per_phase else None
    del G
    torch.cuda.empty_cache()
    sg_ms = None
    if world == 1:
        h, g1 = _single_gpu(*full, V)
        sg = []
        for i in range(args.calls + 1):
            t, _ = _timed(lambda: plc.strongly_connected_components(h, g1, None, None, None, None, False))
            if i:
                sg.append(t)
        sg_ms = sum(sg) / len(sg)
        del g1
    del full
    name, power = _card(local)
    if rank == 0:
        out = {"metric": f"MG SCC RMAT-{args.scale} ef-16 directed, ms per call", "n_gpus": world,
               "grid": f"{groups.R}x{groups.C}", "calls": args.calls, "ms_per_call": sum(ms) / len(ms),
               "ms_min_max": [min(ms), max(ms)], "rounds": rounds, "single_gpu_scc_ms": sg_ms, "parity": par,
               "card": name, "power_limit_w": power,
               "timing": "host clock around the call ending in a device synchronise, max over ranks"}
        if phases is not None:
            out["per_phase"] = phases
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
