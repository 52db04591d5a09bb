"""Multi-GPU Katz, eigenvector centrality and HITS measurement (cugraph_b200.mg.MGGraph), one process per GPU under torchrun:

    torchrun --nproc-per-node N scripts/mg_centrality_bench.py --scale 24 --calls 5

Input: RMAT-`scale` ef-16 (seed 0), directed, unweighted.  Every rank generates the edge list and keeps its share.  Katz uses
alpha = 1 / (1 + the largest in-degree), the default of api.katz_centrality; epsilon is 1e-6 for all three, and at most
200 iterations.
Parity first: on RMAT-16, the MG values must match single-GPU cugraph_katz_centrality / _eigenvector_centrality /
cugraph_hits on rank 0 at the tests' tolerances (Katz rtol 2e-5; eigenvector rtol 2e-3, atol 1e-8; HITS rtol 2e-3,
atol 1e-9); a mismatch ends the run.
Timing: per algorithm one warm-up call (for HITS it builds the block's column-major copy and its sweep layout: its extra
cost over a timed call is reported on its own), then `calls` timed calls, each with a host clock that ends in a device
synchronise, the max over ranks.  ms per call, iterations, ms per iteration.  The single-GPU drivers on the same graph, the
same way, on rank 0 (world size 1 only: the whole graph on one GPU).
Prints one JSON line on rank 0, with the card name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

EPS = dict(katz=1e-6, eigenvector=1e-6, hits=1e-6)
MAX_IT = 200


def _graph(scale, rank, world):
    from cugraph_b200.generators import rmat_edgelist
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    E = src.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    alpha = 1.0 / (1.0 + float(torch.bincount(dst.long()).max().item()))
    return src[lo:hi].clone(), dst[lo:hi].clone(), (src, dst) if rank == 0 else None, alpha


def _gather(verts, vals, V):
    """values of all vertices by id on rank 0 (ids that are not vertices of the graph: 0)"""
    parts = [None] * dist.get_world_size()
    dist.all_gather_object(parts, (verts.cpu(), vals.cpu()))
    out = np.zeros(V)
    for v, x in parts:
        out[v.long().numpy()] = x.double().numpy()
    return out


def _single_gpu(src, dst):
    from cugraph_b200 import pylibcugraph as plc
    h = plc.ResourceHandle()
    g = plc.SGGraph(h, plc.GraphProperties(is_symmetric=False, is_multigraph=True), src, dst, store_transposed=True,
                    renumber=True)
    return h, g


def _sg_calls(h, g, alpha):
    from cugraph_b200 import pylibcugraph as plc
    return dict(katz=lambda: plc.katz_centrality(h, g, None, alpha, 1.0, EPS["katz"], MAX_IT, False),
                eigenvector=lambda: plc.eigenvector_centrality(h, g, EPS["eigenvector"], MAX_IT, False),
                hits=lambda: plc.hits(h, g, EPS["hits"], MAX_IT, None, None, True, False))


def _mg_calls(G, alpha):
    return dict(katz=lambda: G.katz_centrality(alpha, epsilon=EPS["katz"], max_iterations=MAX_IT),
                eigenvector=lambda: G.eigenvector_centrality(epsilon=EPS["eigenvector"], max_iterations=MAX_IT),
                hits=lambda: G.hits(epsilon=EPS["hits"], max_iterations=MAX_IT))


def _iterations(G, name):
    st = {"katz": G.last_katz_stats, "eigenvector": G.last_eigenvector_stats, "hits": G.last_hits_stats}[name]
    return st["iterations"]


def parity(groups, scale=16):
    from cugraph_b200 import mg
    rank, world = dist.get_rank(), dist.get_world_size()
    V = 1 << scale
    s, d, full, alpha = _graph(scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    got = {}
    for name, call in _mg_calls(G, alpha).items():
        out = call()
        got[name] = [_gather(out[0], x, V) for x in out[1:]]
    del G
    if rank != 0:
        return None
    h, g = _single_gpu(*full)
    tol = dict(katz=dict(rtol=2e-5, atol=0.0), eigenvector=dict(rtol=2e-3, atol=1e-8), hits=dict(rtol=2e-3, atol=1e-9))
    res = {"scale": scale}
    ok = True
    for name, call in _sg_calls(h, g, alpha).items():
        out = call()
        ref = [_gather(out[0], x, V) for x in out[1:]]
        good = all(np.allclose(a, b, **tol[name]) for a, b in zip(got[name], ref))
        res[name] = bool(good)
        ok = ok and good
    res["ok"] = ok
    return res


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


def _summary(warm, ms, iters):
    mean = sum(ms) / len(ms)
    return {"ms_per_call": round(mean, 3), "ms_min_max": [round(min(ms), 3), round(max(ms), 3)], "iterations": iters,
            "ms_per_iteration": round(mean / max(iters, 1), 4), "warmup_ms": round(warm, 3)}


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
    os.environ.setdefault("MASTER_PORT", "29533")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    groups = mg.make_groups()
    par = parity(groups)
    ok = torch.tensor([1 if (rank != 0 or par["ok"]) else 0], dtype=torch.int32, device="cuda")
    dist.broadcast(ok, src=0)
    if int(ok.item()) == 0:
        raise SystemExit(f"multi-GPU Katz / eigenvector / HITS do not match single GPU: {par}")
    s, d, full, alpha = _graph(args.scale, rank, world)
    G = mg.MGGraph(s, d, None, groups)
    del s, d
    torch.cuda.empty_cache()
    mg_res = {}
    for name, call in _mg_calls(G, alpha).items():
        warm, _ = _timed(call)                 # HITS: builds the column-major copy and its layout
        ms = [_timed(call)[0] for _ in range(args.calls)]
        mg_res[name] = _summary(warm, ms, _iterations(G, name))
    hw = mg_res["hits"]
    transposed_build_ms = round(hw["warmup_ms"] - hw["ms_per_call"], 3)
    del G
    torch.cuda.empty_cache()
    sg_res = None
    if world == 1:
        h, g = _single_gpu(*full)
        sg_res = {}
        for name, call in _sg_calls(h, g, alpha).items():
            warm, _ = _timed(call)
            ms = [_timed(call)[0] for _ in range(args.calls)]
            sg_res[name] = {"ms_per_call": round(sum(ms) / len(ms), 3), "ms_min_max": [round(min(ms), 3), round(max(ms), 3)]}
        del g
    del full
    name, power = _card(local)
    if rank == 0:
        out = {"metric": f"MG Katz / eigenvector / HITS RMAT-{args.scale} ef-16 directed, ms per call", "n_gpus": world,
               "grid": f"{groups.R}x{groups.C}", "calls": args.calls, "katz_alpha": alpha, "mg": mg_res,
               "hits_first_call_transposed_build_ms": transposed_build_ms, "single_gpu": sg_res, "parity": par,
               "card": name, "power_limit_w": power,
               "timing": "host clock around the call ending in a device synchronise, max over ranks"}
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
