"""Multi-GPU PageRank measurement, plain and personalized (cugraph_b200.mg.MGGraph.pagerank), one process per GPU under
torchrun:

    torchrun --nproc-per-node N scripts/mg_pagerank_bench.py --scale 24 --calls 5

Input: RMAT-`scale` ef-16 (seed 0), directed, unweighted.  Every rank generates the edge list and keeps its share.  Both runs
take 100 iterations at epsilon 0.  The personalized run teleports to 1,024 vertices drawn with seed 1 (among the vertices
of the graph) with values U(0, 1); rank 0 passes them, the others pass None.
Parity first: on RMAT-16, the MG values must match single-GPU cugraph_pagerank_allow_nonconvergence /
cugraph_personalized_pagerank_allow_nonconvergence on rank 0 at the tests' bar (rtol 1e-6, atol 1e-12); a mismatch ends
the run.
Timing: per run one warm-up call, then `calls` timed calls, each with a host clock that ends in a device synchronise, the
max over ranks: ms per call and per iteration.  The two single-GPU entry points on the same graph, the same way, on rank 0
(world size 1 only: the whole graph on one GPU).
Prints one JSON line on rank 0, with the card name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.mg_centrality_bench import _card, _gather, _single_gpu, _timed  # noqa: E402

ALPHA, ITERS, N_PERS = 0.85, 100, 1024
TOL = dict(rtol=1e-6, atol=1e-12)


def _graph(scale, rank, world):
    from cugraph_b200.generators import rmat_edgelist
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    E = src.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    # the personalization: N_PERS vertices of the graph (ids with an edge) drawn with seed 1, values U(0, 1)
    present = torch.unique(torch.cat([src, dst])).cpu().numpy()
    rng = np.random.default_rng(1)
    pick = np.sort(rng.choice(present, size=min(N_PERS, present.size), replace=False))
    pers = (torch.as_tensor(pick.astype(np.int64)).cuda(), torch.as_tensor(rng.uniform(0.0, 1.0, pick.size)).cuda())
    return src[lo:hi].clone(), dst[lo:hi].clone(), (src, dst) if rank == 0 else None, pers


def _mg_calls(G, pers, rank):
    mine = pers if rank == 0 else None
    return dict(plain=lambda: G.pagerank(ALPHA, 0.0, ITERS),
                personalized=lambda: G.pagerank(ALPHA, 0.0, ITERS, personalization=mine))


def _sg_calls(h, g, pers):
    from cugraph_b200 import pylibcugraph as plc
    pv, px = pers[0].to(torch.int32), pers[1].to(torch.float32)
    return dict(plain=lambda: plc.pagerank(h, g, None, None, None, None, ALPHA, 0.0, ITERS, False,
                                           fail_on_nonconvergence=False),
                personalized=lambda: plc.personalized_pagerank(h, g, None, None, None, None, pv, px, ALPHA, 0.0, ITERS,
                                                               False, fail_on_nonconvergence=False))


def parity(groups, scale=16):
    from cugraph_b200 import mg
    rank, world = dist.get_rank(), dist.get_world_size()
    V = 1 << scale
    s, d, full, pers = _graph(scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    got = {}
    for name, call in _mg_calls(G, pers, rank).items():
        v, x, it, _ = call()
        got[name] = (_gather(v, x, V), it)
    del G
    if rank != 0:
        return None
    h, g = _single_gpu(*full)
    res = {"scale": scale}
    ok = True
    for name, call in _sg_calls(h, g, pers).items():
        v, x, _ = call()
        ref = _gather(v, x, V)
        good = bool(np.allclose(got[name][0], ref, **TOL)) and got[name][1] == ITERS
        res[name] = good
        res[name + "_max_rel"] = float(np.max(np.abs(got[name][0] - ref) / np.maximum(np.abs(ref), 1e-30)))
        ok = ok and good
    res["ok"] = ok
    return res


def _summary(warm, ms):
    mean = sum(ms) / len(ms)
    return {"ms_per_call": round(mean, 3), "ms_min_max": [round(min(ms), 3), round(max(ms), 3)],
            "ms_per_iteration": round(mean / ITERS, 4), "warmup_ms": round(warm, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--calls", type=int, default=5)
    args = ap.parse_args()
    from cugraph_b200 import mg
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29535")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    groups = mg.make_groups()
    par = parity(groups)
    ok = torch.tensor([1 if (rank != 0 or par["ok"]) else 0], dtype=torch.int32, device="cuda")
    dist.broadcast(ok, src=0)
    if int(ok.item()) == 0:
        raise SystemExit(f"multi-GPU PageRank does not match single GPU: {par}")
    s, d, full, pers = _graph(args.scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    del s, d
    torch.cuda.empty_cache()
    mg_res = {}
    for name, call in _mg_calls(G, pers, rank).items():
        warm, _ = _timed(call)
        ms = [_timed(call)[0] for _ in range(args.calls)]
        mg_res[name] = _summary(warm, ms)
    del G
    torch.cuda.empty_cache()
    sg_res = None
    if world == 1:
        h, g = _single_gpu(*full)
        sg_res = {}
        for name, call in _sg_calls(h, g, pers).items():
            warm, _ = _timed(call)
            ms = [_timed(call)[0] for _ in range(args.calls)]
            sg_res[name] = _summary(warm, ms)
        del g
    del full
    name, power = _card(local)
    if rank == 0:
        out = {"metric": f"MG PageRank RMAT-{args.scale} ef-16 directed, {ITERS} iterations, ms per call", "n_gpus": world,
               "grid": f"{groups.R}x{groups.C}", "calls": args.calls, "personalization_vertices": int(pers[0].numel()),
               "mg": mg_res, "single_gpu": sg_res, "parity": par, "card": name, "power_limit_w": power,
               "timing": "host clock around the call ending in a device synchronise, max over ranks"}
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
