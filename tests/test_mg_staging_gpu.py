"""MGGraph's construction options on the GPU.

- cugraph_b200_block_stage_edges against the numpy restatement (tests/mg_staging_ref.py), unweighted / float32 / float64.
- Every rank of a 1x2, 2x1, 2x2 and 4x2 grid on ONE GPU in one process (tests/mg_world.py) against the single-GPU
  constructor with the same options, on the hand-made graph with isolated vertices and on RMAT-14 / RMAT-16: degrees,
  SSSP and BFS bit-exact, PageRank within 1e-6, WCC from one-direction input with symmetrize.
- A world-size-1 NCCL process group (the real collectives and stream ordering), and 2 / 4 GPUs over NCCL (skipped when
  fewer GPUs are visible), against the numpy restatement."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_staging_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.test_mg_staging_cpu import CENTRALITY, _check, _runs, _same  # noqa: E402

pytestmark = pytest.mark.gpu

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]


@pytest.mark.parametrize("wdtype", [None, np.float32, np.float64], ids=["unweighted", "f32", "f64"])
def test_block_stage_edges_against_numpy_on_gpu(wdtype):
    rng = np.random.default_rng(12)
    for dm in (False, True):
        for sym in (False, True):
            for n_rows, n_cols, n in ((50, 70, 3000), (3000, 700, 40000)):
                rows, cols, rev, w = refs.random_block(rng, n_rows, n_cols, n, wdtype)
                _same(refs.stage_block(rows, cols, rev, w, n_rows, n_cols, dm, sym),
                      refs.stage_block_np(rows, cols, rev, w, dm, sym))


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_staging_hand_graph_on_one_gpu(monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, w, iso = refs.hand_graph()
    for opts in refs.OPTIONS:
        runs = _runs(True, [0, 8, 40]) + [("wcc", {})] * opts["symmetrize"]
        for split in refs.vertex_splits(iso, s, world):
            _check(s, d, w.astype(np.float32), world, opts, split, runs, "cuda", partition=("wcc",))
        _check(s, d, None, world, opts, [iso] + [None] * (world - 1), _runs(False, [2]) + CENTRALITY, "cuda")


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_staging_rmat_on_one_gpu(monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    for scale, wdtype in ((14, np.float32), (16, np.float64)):
        s, d, w, V = refs.rmat_graph(scale, wdtype=wdtype)
        extra = np.arange(V, V + 6, dtype=np.int32)
        for opts in (dict(drop_multi_edges=True), dict(symmetrize=True),
                     dict(drop_self_loops=True, drop_multi_edges=True, symmetrize=True)):
            runs = [("pagerank", dict(alpha=0.85, epsilon=0.0, max_iterations=30)), ("sssp", dict(source=int(s[0]))),
                    ("bfs", dict(source=int(d[7])))] + [("wcc", {})] * opts.get("symmetrize", False)
            _check(s, d, w, world, opts, [extra[:4]] + [None] * (world - 2) + [extra[2:]], runs, "cuda", partition=("wcc",))


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _nccl_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    s, d, w, iso = refs.hand_graph()
    s_, d_, w_ = mg_world.share(rank, world, s, d, w)
    g = mg.MGGraph(torch.as_tensor(s_).cuda(), torch.as_tensor(d_).cuda(), torch.as_tensor(w_).cuda(),
                   vertices=torch.as_tensor(iso).cuda() if rank == 0 else None, drop_self_loops=True, drop_multi_edges=True,
                   symmetrize=True)
    v, din, dout = mg.degrees(g)
    _, dist, _ = mg.sssp(g, 0, compute_predecessors=False)
    return v.cpu().numpy(), din.cpu().numpy(), dout.cpu().numpy(), dist.cpu().numpy()


def _run_nccl(world):
    import oracle
    res = mg_procs.run(_nccl_worker, world, backend="nccl", timeout=600)
    s, d, w, iso = refs.hand_graph()
    opts = dict(drop_self_loops=True, drop_multi_edges=True, symmetrize=True)
    verts, (S, D, W) = refs.stage_graph_np(s, d, w, iso, **opts)
    din, dout = refs.degrees_np(verts, S, D)
    want, _ = oracle.sssp(S, D, W, int(verts.max()) + 1, 0, cutoff=None, use_float=False)
    got = {}
    for v, a, b, x in res:
        for k in range(v.size):
            got[int(v[k])] = (a[k], b[k], x[k])
    assert sorted(got) == verts.tolist()
    for i, v in enumerate(verts.tolist()):
        assert got[v][:2] == (din[i], dout[i])
        assert got[v][2] == min(want[v], np.finfo(np.float64).max)


def test_mg_staging_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_staging_multi_gpu(world):
    _run_nccl(world)
