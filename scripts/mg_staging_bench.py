"""Multi-GPU graph construction with the staging options (cugraph_b200.mg.MGGraph), one process per GPU under torchrun:

    torchrun --nproc-per-node N scripts/mg_staging_bench.py --scale 24 --calls 3

Input: RMAT-`scale` ef-16 (seed 0), one direction, weights U(0, 1) in float32 (seed 1).  Every rank generates the edge list
and keeps its share.  Three constructions: the default (the edges as given); symmetrize=True; symmetrize=True with
drop_multi_edges=True.  Per construction one warm-up, then `calls` timed constructions, each with a host clock that ends in
a device synchronise, the max over ranks; and the peak device memory of one more construction, the max over ranks, from
both allocators that hold it:
  torch: torch.cuda.max_memory_allocated / max_memory_reserved after a reset (the input edge list, the shuffle's and the
    partition's tensors);
  library: the high-water marks of used and of reserved (backing) memory of the device's default memory pool, reset before
    the construction (cuMemPoolGetAttribute; the library allocates its staging sorts, CUB scratch and the block's own
    layouts there with cudaMallocAsync, which torch's counters do not see).
The sum of the two reserved peaks bounds what the construction occupies on the card (the two peaks need not coincide).
Prints one JSON line on rank 0, with the card name and power limit read in the same run."""
from __future__ import annotations

import argparse
import ctypes
import gc
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.mg_centrality_bench import _card, _timed  # noqa: E402

CASES = {"default": {}, "symmetrize": dict(symmetrize=True),
         "symmetrize+drop_multi_edges": dict(symmetrize=True, drop_multi_edges=True)}


class _LibraryPool:
    """high-water marks of the device's default memory pool (CUDA driver API), where the library's cudaMallocAsync
    allocations live"""
    RESERVED_HIGH, USED_CURRENT, USED_HIGH = 6, 7, 8   # CUmemPool_attribute

    def __init__(self, device):
        self.cu = ctypes.CDLL("libcuda.so.1")
        dev, self.pool = ctypes.c_int(), ctypes.c_void_p()
        self._ok(self.cu.cuDeviceGet(ctypes.byref(dev), device))
        self._ok(self.cu.cuDeviceGetDefaultMemPool(ctypes.byref(self.pool), dev))

    @staticmethod
    def _ok(code):
        if code != 0:
            raise RuntimeError(f"CUDA driver call failed: {code}")

    def get(self, attr):
        v = ctypes.c_uint64()
        self._ok(self.cu.cuMemPoolGetAttribute(self.pool, attr, ctypes.byref(v)))
        return v.value

    def reset(self):
        for attr in (self.RESERVED_HIGH, self.USED_HIGH):
            self._ok(self.cu.cuMemPoolSetAttribute(self.pool, attr, ctypes.byref(ctypes.c_uint64(0))))


def _edges(scale, rank, world):
    from cugraph_b200.generators import rmat_edgelist
    src, dst = rmat_edgelist(scale, 16 << scale, seed=0)
    E = src.numel()
    lo, hi = rank * E // world, (rank + 1) * E // world
    g = torch.Generator(device="cuda").manual_seed(1)
    w = torch.rand(E, generator=g, device="cuda", dtype=torch.float32)
    return src[lo:hi].clone(), dst[lo:hi].clone(), w[lo:hi].clone()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=24)
    ap.add_argument("--calls", type=int, default=3)
    args = ap.parse_args()
    from cugraph_b200 import mg
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", str(rank)))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29536")
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", local))
    groups = mg.make_groups()
    s, d, w = _edges(args.scale, rank, world)
    pool = _LibraryPool(local)
    res = {}
    for name, opts in CASES.items():
        def build():
            return mg.MGGraph(s, d, w, groups, **opts)
        warm, G = _timed(build)
        edges = torch.tensor([G.num_edges_local], dtype=torch.int64, device="cuda")
        dist.all_reduce(edges)
        del G
        ms = []
        for _ in range(args.calls):
            t, G = _timed(build)
            ms.append(t)
            del G
        gc.collect()
        torch.cuda.empty_cache()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        lib_before = pool.get(pool.USED_CURRENT)
        pool.reset()
        G = build()
        torch.cuda.synchronize()
        peak = torch.tensor([torch.cuda.max_memory_allocated(), torch.cuda.max_memory_reserved(), pool.get(pool.USED_HIGH),
                             pool.get(pool.RESERVED_HIGH), lib_before], dtype=torch.int64, device="cuda")
        dist.all_reduce(peak, op=dist.ReduceOp.MAX)
        del G
        gc.collect()
        torch.cuda.empty_cache()
        gib = [round(int(x) / 2**30, 3) for x in peak.tolist()]
        res[name] = {"ms_per_construction": round(sum(ms) / len(ms), 1), "ms_min_max": [round(min(ms), 1), round(max(ms), 1)],
                     "warmup_ms": round(warm, 1), "torch_peak_allocated_gib": gib[0], "torch_peak_reserved_gib": gib[1],
                     "library_pool_peak_used_gib": gib[2], "library_pool_peak_reserved_gib": gib[3],
                     "library_pool_used_before_gib": gib[4], "card_bound_gib": round(gib[1] + gib[3], 3),
                     "stored_edges": int(edges.item())}
    name, power = _card(local)
    if rank == 0:
        out = {"metric": f"MGGraph construction RMAT-{args.scale} ef-16, float32 weights, ms per construction",
               "n_gpus": world, "grid": f"{groups.R}x{groups.C}", "input_edges": 16 << args.scale, "calls": args.calls,
               "cases": res, "card": name, "power_limit_w": power,
               "timing": "host clock around the construction ending in a device synchronise, max over ranks"}
        print(json.dumps(out), flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
