"""Multi-GPU BFS from a set of sources and multi-GPU extract_paths on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running MGGraph.bfs and MGGraph.extract_paths: grids
  1x2, 2x1, 2x2 and 4x2 on directed RMAT-14 and RMAT-16 with sources split over the ranks and a rank without
  destinations, and on a forest with forced predecessors, where the rows are bit-identical to single-GPU
  cugraph_extract_paths.  Distances bit-exact against the oracle and single-GPU cugraph_bfs from the same sources,
  predecessors by the reference's predicate, paths against a numpy restatement of single GPU's walk.
- A world-size-1 NCCL process group (the 1x1 grid): the real collectives and the real stream ordering on the device.
- 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_paths_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402

pytestmark = pytest.mark.gpu


def _inputs(s, d, world, seed, n_sources=16, n_dests=3000):
    rng = np.random.default_rng(seed)
    ids = np.unique(np.concatenate([s, d]))
    srcs = rng.choice(np.flatnonzero(np.bincount(s) > 0), n_sources, replace=False).astype(np.int32)
    pool = np.concatenate([rng.choice(ids, n_dests), srcs, refs.not_vertices(s, d)]).astype(np.int32)
    rng.shuffle(pool)
    dests = refs.split(pool, world - 1, rng) + [np.zeros(0, np.int32)] if world > 1 else [pool]
    return srcs, refs.split(srcs, world, rng), dests


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_paths_simulated_on_one_gpu(monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    for scale in (14, 16):
        s, d = refs.rmat_graph(scale)
        srcs, sources, dests = _inputs(s, d, world, scale)
        res = refs.mg_bfs_paths(s, d, world, sources, dests, device="cuda", repeat=True)
        got_d = refs.check_bfs(s, d, res, srcs)
        refs.check_paths(res, dests)
        sg_dist, _ = refs.single_gpu_paths(s, d, srcs, dests[0])
        ids, remap = mg_world.present(s, d, sg_dist.size)
        assert np.array_equal(sg_dist[ids], got_d)                     # single-GPU cugraph_bfs from the same sources
    res = refs.mg_bfs_paths(s, d, world, sources, dests, depth_limit=2, device="cuda")
    refs.check_bfs(s, d, res, srcs, depth_limit=2)
    refs.check_paths(res, dests)
    s, d, roots, unreached = refs.forced_graph(n_tree=5000, n_roots=9, n_cycle=300)
    pool = np.concatenate([np.unique(np.concatenate([s, d])), roots, refs.not_vertices(s, d)]).astype(np.int32)
    dests = refs.split(pool, world, np.random.default_rng(1))
    res = refs.mg_bfs_paths(s, d, world, refs.split(roots, world, np.random.default_rng(2)), dests, device="cuda")
    refs.check_bfs(s, d, res, roots)
    paths, _ = refs.check_paths(res, dests)
    _, sg_paths = refs.single_gpu_paths(s, d, roots, pool)
    assert np.array_equal(np.concatenate([r["paths"] for r in res]), sg_paths)


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _nccl_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    s, d = refs.rmat_graph(14)
    srcs, sources, dests = _inputs(s, d, world, 3)
    E = s.size
    lo, hi = rank * E // world, (rank + 1) * E // world
    g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda())
    v, dist, pred = mg.bfs(g, torch.as_tensor(sources[rank]).cuda())
    paths, length = mg.extract_paths(g, dist, pred, torch.as_tensor(dests[rank]).cuda())
    one = mg.bfs(g, int(srcs[0]))
    one_t = mg.bfs(g, torch.tensor([int(srcs[0])], dtype=torch.int32).cuda())
    same = all(torch.equal(a, b) for a, b in zip(one, one_t))
    return dict(v=v.cpu().numpy(), dist=dist.cpu().numpy(), pred=pred.cpu().numpy(), paths=paths.cpu().numpy(),
                length=length, rounds=g.last_paths_stats["rounds"], same=same)


def _run_nccl(world):
    res = mg_procs.run(_nccl_worker, world, backend="nccl", timeout=600)
    s, d = refs.rmat_graph(14)
    srcs, _, dests = _inputs(s, d, world, 3)
    refs.check_bfs(s, d, res, srcs)
    refs.check_paths(res, dests)
    assert all(r["same"] for r in res)


def test_mg_paths_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_paths_multi_gpu(world):
    _run_nccl(world)
