"""Multi-GPU multi-source BFS on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running MGGraph.multi_source_bfs: grids 1x2, 2x1, 2x2
  and 4x2, the four schedules and the graphs of tests/mg_bfs_direction_ref.py (RMAT-12), 1, 63, 64, 65 and 130 sources
  with a duplicate, depth limits 0, 1, 3 and none, with every check of tests/mg_ms_bfs_ref.py; the distance rows also
  against single-GPU cugraph_b200_multi_source_bfs on the same edge list.
- The five entry points against numpy on one block on the device.
- A world-size-1 NCCL process group (the 1x1 grid), and 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible):
  every schedule against the oracle and MGGraph.bfs, and a repeated call."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_bfs_direction_ref as dref  # noqa: E402
from tests import mg_ms_bfs_ref as ref  # noqa: E402
from tests import mg_paths_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.test_mg_multi_source_bfs_cpu import check_block_steps, check_owner_steps  # noqa: E402

pytestmark = pytest.mark.gpu

SIZES = dict(path=300, grid=30, core=12, tail=150, clique=100, components=300)
LIMITS = (-1, 0, 1, 3)


def _sizes():
    from cugraph_b200 import _capi
    from tests.test_traversal_shapes_gpu import EMU_SIZES
    return dict(EMU_SIZES, path=30, grid=6, tail=12, components=30) if _capi.emulated() else SIZES


def _scale():
    from cugraph_b200 import _capi
    return 8 if _capi.emulated() else 12


def single_gpu_rows(s, d, sources, symmetric):
    """cugraph_b200_multi_source_bfs on the single-GPU graph of the edges: distances [n, V] by vertex id (-5 for ids that
    are not vertices)"""
    import torch
    from cugraph_b200.traversal import multi_source_bfs
    from tests.gpu_util import make_graph
    h, g = make_graph(s, d, symmetric=symmetric)
    dist, _, verts = multi_source_bfs(h, g, torch.as_tensor(np.asarray(sources, np.int32)).cuda(), 0, False)
    out = np.full((len(sources), int(max(s.max(), d.max())) + 1), -5, np.int64)
    out[:, verts.cpu().numpy()] = dist.cpu().numpy()
    return out


@pytest.mark.parametrize("schedule", list(dref.SCHEDULES))
@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_multi_source_bfs_simulated_on_one_gpu(monkeypatch, R, Cc, schedule):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    dref.set_knobs(monkeypatch, dref.SCHEDULES[schedule][1])
    gi, si = [(1, 2), (2, 1), (2, 2), (4, 2)].index((R, Cc)), list(dref.SCHEDULES).index(schedule)
    rng = np.random.default_rng(gi * 10 + si)
    for i, case in enumerate(dref.cases(_sizes(), _scale())):
        n = ref.SOURCE_COUNTS[(i + gi + si) % len(ref.SOURCE_COUNTS)]
        ref.run_case(case, world, schedule, n, LIMITS[(i + 2 * gi + si) % len(LIMITS)], rng, device="cuda")


def _rows_worker(rank, world, s, d, sources):
    import torch
    g = mg_world.graph(rank, world, s, d, device="cuda")
    v, dist, _ = g.multi_source_bfs(torch.as_tensor(sources).cuda(), compute_predecessors=False)
    return dict(v=v.cpu().numpy(), dist=dist.cpu().numpy())


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 2)], ids=["1x2", "2x2"])
def test_mg_multi_source_bfs_matches_single_gpu(monkeypatch, R, Cc):
    """the distance rows equal single GPU's multi-source BFS on the same edge list, gathered by vertex id"""
    world = mg_world.grid_world(monkeypatch, R, Cc)
    rng = np.random.default_rng(R * 10 + Cc)
    s, d = refs.rmat_graph(_scale() + 2)
    for gs, gd, sym in ((s, d, False), (np.concatenate([s, d]), np.concatenate([d, s]), True)):
        srcs = rng.choice(np.unique(np.concatenate([gs, gd])), 100).astype(np.int32)
        res = mg_world.run(world, _rows_worker, gs, gd, srcs)
        want = single_gpu_rows(gs, gd, srcs, sym)
        for r in res:
            assert np.array_equal(want[:, r["v"]], r["dist"])


def test_ms_bfs_entry_points_against_numpy_on_gpu():
    rng = np.random.default_rng(7)
    n_rows, n_cols, m = 3000, 5000, 40000
    rows = rng.integers(0, n_rows, m).astype(np.int32)
    cols = rng.integers(0, n_cols, m).astype(np.int32)
    rows[: m // 10] = 17                                  # a dense row: the warp kernels
    cols[m // 10: m // 5] = 11                            # a hub column: the merge-path advance splits its edges
    b = dref.Block(rows, cols, n_rows, n_cols, device="cuda")
    try:
        check_block_steps(b, rows, cols, n_rows, n_cols, rng, "cuda",
                          ((1000, 3, 2, 64, 0.01, 0.2), (3000, 1, 0, 20, 0.6, 0.0), (750, 4, 1, 64, 0.9, 0.95)))
    finally:
        b.close()
    check_owner_steps(rng, "cuda", ((1, 3000, 3000, 64, 3, True), (4, 1000, 900, 17, 2, False), (2, 100, 0, 1, 1, True)))


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _nccl_worker(rank, world, s, d, sources):
    import torch
    from cugraph_b200 import mg
    E = s.size
    lo, hi = rank * E // world, (rank + 1) * E // world
    out = {}
    for name, (do, knobs) in dref.SCHEDULES.items():
        for k in dref.KNOBS:
            os.environ.pop(k, None)
        os.environ.update(knobs)
        g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda())
        src = torch.as_tensor(sources).cuda()
        v, dist, pred = mg.multi_source_bfs(g, src, direction_optimizing=do)
        _, d2, p2 = mg.multi_source_bfs(g, src, direction_optimizing=do)
        _, d1, p1 = g.bfs(int(sources[-1]))
        out[name] = dict(v=v.cpu().numpy(), dist=dist.cpu().numpy(), pred=pred.cpu().numpy(), n_local=g.part.n_local,
                         same=bool(torch.equal(d2, dist) and torch.equal(p2, pred) and torch.equal(dist[-1], d1)
                                   and torch.equal(pred[-1], p1)), stats=g.last_ms_bfs_stats)
        del g
    return out


def _run_nccl(world):
    s, d = refs.rmat_graph(12)
    rng = np.random.default_rng(world)
    for gs, gd in ((s, d), (np.concatenate([s, d]), np.concatenate([d, s]))):
        srcs = rng.choice(np.unique(np.concatenate([gs, gd])), 70).astype(np.int32)
        out = mg_procs.run(_nccl_worker, world, gs, gd, srcs, backend="nccl", timeout=600)
        for name in dref.SCHEDULES:
            res = [o[name] for o in out]
            ecc = ref.check_rows(gs, gd, res, srcs)
            st = res[0]["stats"]
            assert all(r["same"] and r["stats"] == st for r in res), name
            assert st["levels"] == ref.expected_levels(ecc, -1) and st["batches"] == 2, (name, st)
            assert name != "top_down" or st["bottom_up"] == 0, (name, st)


def test_mg_multi_source_bfs_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_multi_source_bfs_multi_gpu(world):
    _run_nccl(world)
