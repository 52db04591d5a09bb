"""Multi-GPU BFS top-down and direction-optimising on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running MGGraph.bfs(direction_optimizing=...): grids
  1x2, 2x1, 2x2 and 4x2 on the graphs of tests/mg_bfs_direction_ref.py (directed and symmetrised RMAT-14, a path with
  int64 external ids, a grid with edges removed, a lollipop, a union of small components, a forest with forced
  predecessors) in the four schedules of that module, with every check there; on the forest, predecessors bit-identical
  to single-GPU cugraph_bfs.
- The default schedule on a symmetric RMAT-16 runs both directions, the same number of levels each as cugraph_bfs's
  trace.
- cugraph_b200_block_bfs_push against numpy on one block on the device.
- A world-size-1 NCCL process group (the 1x1 grid), and 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible):
  every schedule against the oracle and a repeated call."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_bfs_direction_ref as ref  # noqa: E402
from tests import mg_paths_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402

pytestmark = pytest.mark.gpu

# every level of a traversal is a round of collectives: the path and the grid are kept to a few hundred levels
SIZES = dict(path=600, grid=60, core=12, tail=300, clique=200, components=500)


def _scale():
    from cugraph_b200 import _capi
    return 8 if _capi.emulated() else 14


def _sizes():
    from cugraph_b200 import _capi
    from tests.test_traversal_shapes_gpu import EMU_SIZES
    return dict(EMU_SIZES, path=40, grid=8, tail=20, components=40) if _capi.emulated() else SIZES


@pytest.mark.parametrize("schedule", list(ref.SCHEDULES))
@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_bfs_direction_simulated_on_one_gpu(monkeypatch, R, Cc, schedule):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    ref.set_knobs(monkeypatch, ref.SCHEDULES[schedule][1])
    rng = np.random.default_rng(R * 10 + Cc)
    for case in ref.cases(_sizes(), _scale()):
        res = ref.run_case(case, world, schedule, rng, device="cuda")
        if case.name == "forced":
            sg_d, sg_p = ref.single_gpu_bfs(case.s, case.d, case.sources, False, False)
            vids, dist, pred = refs.gather(res)
            assert np.array_equal(sg_d[vids], dist) and np.array_equal(sg_p[vids], pred), schedule


def _schedule_worker(rank, world, s, d, src):
    g = mg_world.graph(rank, world, s, d, device="cuda")
    v, dist, _ = g.bfs(src, direction_optimizing=True)
    return dict(stats=g.last_bfs_stats, v=v.cpu().numpy(), dist=dist.cpu().numpy())


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 2)], ids=["1x2", "2x2"])
def test_mg_bfs_default_schedule_is_single_gpu_schedule(monkeypatch, capfd, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    ref.set_knobs(monkeypatch, {})
    s, d = refs.rmat_graph(_scale() + 2)
    s, d = np.concatenate([s, d]), np.concatenate([d, s])
    deg = np.bincount(s)
    hub = int(deg.argmax())
    for src in [hub] + np.flatnonzero((deg >= 5) & (deg <= 50))[:2].tolist():
        res = mg_world.run(world, _schedule_worker, s, d, src)
        monkeypatch.setenv("CUGRAPH_B200_BFS_TRACE", "1")
        capfd.readouterr()
        sg_d, _ = ref.single_gpu_bfs(s, d, [src], True, True)
        td, bu = ref.trace_directions(capfd.readouterr().err)
        monkeypatch.delenv("CUGRAPH_B200_BFS_TRACE")
        assert bu > 0 and (td > 0 or src == hub), src
        for r in res:
            assert (r["stats"]["top_down"], r["stats"]["bottom_up"]) == (td, bu), (src, r["stats"])
            assert np.array_equal(sg_d[r["v"]], r["dist"])


def test_block_bfs_push_against_numpy_on_gpu():
    import torch
    rng = np.random.default_rng(7)
    n_rows, n_cols, m = 30000, 50000, 400000
    rows = rng.integers(0, n_rows, m).astype(np.int32)
    cols = rng.integers(0, n_cols, m).astype(np.int32)
    cols[: m // 10] = 11                                  # a hub column: the merge-path advance splits its edges
    b = ref.Block(rows, cols, n_rows, n_cols, device="cuda")
    try:
        for maxpart, grid_cols, grid_c, pf, pv in ((20000, 3, 2, 0.01, 0.2), (50000, 1, 0, 0.6, 0.0), (7000, 4, 1, 1.0, 0.95)):
            frontier = (rng.random(n_cols) < pf).astype(np.uint8)
            visited = (rng.random(n_rows) < pv).astype(np.uint8)
            cand = torch.full((n_rows,), 77, dtype=torch.int64, device="cuda")
            b.call("cugraph_b200_block_bfs_push", torch.as_tensor(frontier).cuda(), torch.as_tensor(visited).cuda(), maxpart,
                   grid_cols, grid_c, cand)
            torch.cuda.synchronize()
            want = ref.push_reference(rows, cols, n_rows, frontier, visited, maxpart, grid_cols, grid_c)
            assert np.array_equal(cand.cpu().numpy(), want)
    finally:
        b.close()


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _nccl_worker(rank, world, s, d, sources):
    import torch
    from cugraph_b200 import mg
    E = s.size
    lo, hi = rank * E // world, (rank + 1) * E // world
    out = {}
    for name, (do, knobs) in ref.SCHEDULES.items():
        for k in ref.KNOBS:
            os.environ.pop(k, None)
        os.environ.update(knobs)
        g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda())
        src = torch.as_tensor(sources[rank]).cuda()
        v, dist, pred = mg.bfs(g, src, direction_optimizing=do)
        again = mg.bfs(g, src, direction_optimizing=do)[2]
        out[name] = dict(v=v.cpu().numpy(), dist=dist.cpu().numpy(), pred=pred.cpu().numpy(),
                         same=bool(torch.equal(again, pred)), stats=g.last_bfs_stats)
        del g
    return out


def _run_nccl(world):
    s, d = refs.rmat_graph(14)
    rng = np.random.default_rng(world)
    for gs, gd in ((s, d), (np.concatenate([s, d]), np.concatenate([d, s]))):
        srcs = rng.choice(np.flatnonzero(np.bincount(gs) > 0), 8, replace=False).astype(np.int32)
        out = mg_procs.run(_nccl_worker, world, gs, gd, refs.split(srcs, world, rng), backend="nccl", timeout=600)
        for name in ref.SCHEDULES:
            res = [o[name] for o in out]
            refs.check_bfs(gs, gd, res, srcs)
            st = res[0]["stats"]
            assert all(r["same"] and r["stats"] == st for r in res), name
            assert (name != "top_down" or st["bottom_up"] == 0) and (name != "bottom_up" or st["top_down"] == 0), (name, st)


def test_mg_bfs_direction_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_bfs_direction_multi_gpu(world):
    _run_nccl(world)
