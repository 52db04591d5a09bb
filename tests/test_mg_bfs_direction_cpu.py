"""Multi-GPU BFS top-down and direction-optimising on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running MGGraph.bfs(direction_optimizing=...): grids 1x2, 2x1,
  2x2 and 4x2; directed and symmetrised RMAT-8, a path with int64 external ids, a grid with edges removed, a lollipop, a
  union of small components and a forest with forced predecessors (tests/mg_bfs_direction_ref.py); four schedules:
  top-down, direction-optimising with the default knobs, with knobs that keep every level bottom-up and with knobs that
  switch at almost every level.  Each run: distances bit-exact against the oracle, predecessors by the reference's
  predicate, depth limits 1, D / 2, D and D + 1, extract_paths on the result, a repeated call with identical predecessors,
  the level counts of last_bfs_stats; on the forced forest, predecessors bit-identical to single-GPU cugraph_bfs.
- The schedule on a symmetric RMAT is single GPU's: the same top-down / bottom-up level counts as cugraph_bfs's trace.
- cugraph_b200_block_bfs_push against numpy on one block, with its argument errors; cugraph_b200_bfs_bottom_up against
  a table of Beamer's rule, with the default and with set knobs.
- World sizes 2 and 4 over gloo, directed and symmetric, every schedule."""
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
from tests.emu_py import surface  # noqa: E402, F401
from tests.test_traversal_shapes_gpu import EMU_SIZES  # noqa: E402

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]
SIZES = dict(EMU_SIZES, path=40, grid=8, tail=20, components=40)   # every level is a round of collectives


@pytest.mark.parametrize("schedule", list(ref.SCHEDULES))
@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_bfs_direction_emulated(surface, monkeypatch, R, Cc, schedule):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    ref.set_knobs(monkeypatch, ref.SCHEDULES[schedule][1])
    rng = np.random.default_rng(R * 10 + Cc)
    for case in ref.cases(SIZES, 8):
        res = ref.run_case(case, world, schedule, rng)
        if case.name == "forced":   # one possible predecessor per vertex: single GPU's, bit for bit
            sg_d, sg_p = ref.single_gpu_bfs(case.s, case.d, case.sources, False, False)
            vids, dist, pred = refs.gather(res)
            assert np.array_equal(sg_d[vids], dist) and np.array_equal(sg_p[vids], pred), schedule


def _schedule_worker(rank, world, s, d, src):
    g = mg_world.graph(rank, world, s, d)
    g.bfs(src, direction_optimizing=True)
    return g.last_bfs_stats


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 2)], ids=["1x2", "2x2"])
def test_mg_bfs_default_schedule_is_single_gpu_schedule_emulated(surface, monkeypatch, capfd, R, Cc):
    """default knobs on a symmetric RMAT: from a low-degree source the first level runs top-down and the next ones
    bottom-up, and every source gives the same number of levels in each direction as cugraph_bfs"""
    world = mg_world.grid_world(monkeypatch, R, Cc)
    ref.set_knobs(monkeypatch, {})
    s, d = refs.rmat_graph(10)
    s, d = np.concatenate([s, d]), np.concatenate([d, s])
    deg = np.bincount(s)
    hub = int(deg.argmax())
    for src in [hub] + np.flatnonzero((deg >= 5) & (deg <= 50))[:2].tolist():
        stats = mg_world.run(world, _schedule_worker, s, d, src)
        monkeypatch.setenv("CUGRAPH_B200_BFS_TRACE", "1")
        capfd.readouterr()
        ref.single_gpu_bfs(s, d, [src], True, True)
        td, bu = ref.trace_directions(capfd.readouterr().err)
        monkeypatch.delenv("CUGRAPH_B200_BFS_TRACE")
        assert bu > 0 and (td > 0 or src == hub), src     # the hub's edges alone switch the first level
        for st in stats:
            assert (st["top_down"], st["bottom_up"]) == (td, bu), (src, st)


# ---------------------------------------------------------------------------------------------------- the entry points
def _block(rng, n_rows, n_cols, m):
    rows = rng.integers(0, n_rows, m).astype(np.int32)
    cols = rng.integers(0, n_cols, m).astype(np.int32)
    rows[: m // 8] = 3          # a dense row (the push copy's hub columns are the dense part)
    cols[m // 8: m // 4] = 5
    return rows, cols, ref.Block(rows, cols, n_rows, n_cols)


def test_block_bfs_push_against_numpy_emulated(surface):
    import torch
    rng = np.random.default_rng(4)
    n_rows, n_cols = 700, 900
    rows, cols, b = _block(rng, n_rows, n_cols, 6000)
    try:
        for maxpart, grid_cols, grid_c, pf, pv in ((300, 3, 1, 0.05, 0.3), (450, 2, 0, 0.5, 0.0), (900, 1, 0, 0.0, 0.5),
                                                   (100, 4, 3, 1.0, 0.9)):
            frontier = (rng.random(n_cols) < pf).astype(np.uint8)
            visited = (rng.random(n_rows) < pv).astype(np.uint8)
            cand = torch.full((n_rows + 3,), 77, dtype=torch.int64)        # stale values and a longer array
            b.call("cugraph_b200_block_bfs_push", torch.as_tensor(frontier), torch.as_tensor(visited), maxpart, grid_cols,
                   grid_c, cand)
            want = ref.push_reference(rows, cols, n_rows, frontier, visited, maxpart, grid_cols, grid_c)
            assert np.array_equal(cand.numpy()[:n_rows], want)
            assert (cand.numpy()[n_rows:] == 77).all()
            # the pull step finds a frontier source of the same rows
            pull = torch.full((n_rows,), 77, dtype=torch.int64)
            b.call("cugraph_b200_block_bfs_pull", torch.as_tensor(frontier), torch.as_tensor(visited), maxpart, grid_cols,
                   grid_c, pull)
            assert np.array_equal(pull.numpy() >= 0, want >= 0)
    finally:
        b.close()


def test_block_bfs_push_errors_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    rng = np.random.default_rng(5)
    n_rows, n_cols = 40, 60
    _, _, b = _block(rng, n_rows, n_cols, 300)
    u8 = torch.uint8
    f, v, c = torch.zeros(n_cols, dtype=u8), torch.zeros(n_rows, dtype=u8), torch.zeros(n_rows, dtype=torch.int64)
    base = dict(f=f, v=v, c=c, maxpart=20, grid_cols=3, grid_c=1)
    cases = {"frontier dtype": dict(f=f.int()), "visited dtype": dict(v=v.long()), "cand dtype": dict(c=c.int()),
             "short frontier": dict(f=f[:-1]), "short visited": dict(v=v[:-1]), "short cand": dict(c=c[:-1]),
             "maxpart": dict(maxpart=0), "grid_cols": dict(grid_cols=0), "grid_c": dict(grid_c=3),
             "negative grid_c": dict(grid_c=-1)}
    want = {"frontier dtype": "byte flags", "visited dtype": "byte flags", "cand dtype": "cand must be INT64",
            "short frontier": "shorter", "short visited": "shorter", "short cand": "shorter", "maxpart": "bad grid position",
            "grid_cols": "bad grid position", "grid_c": "bad grid position", "negative grid_c": "bad grid position"}
    try:
        for name, kw in cases.items():
            a = dict(base, **kw)
            for fn in ("cugraph_b200_block_bfs_push", "cugraph_b200_block_bfs_pull"):   # the same checks, the same messages
                with pytest.raises(_capi.CugraphError) as e:
                    b.call(fn, a["f"], a["v"], a["maxpart"], a["grid_cols"], a["grid_c"], a["c"])
                assert e.value.code == _capi.INVALID_INPUT and want[name] in str(e.value), (fn, name, str(e.value))
        b.call("cugraph_b200_block_bfs_push", f, v, 20, 3, 2, c)   # the block still works
        assert (c.numpy() == -1).all()
    finally:
        b.close()


def _bottom_up_table():
    rng = np.random.default_rng(6)
    rows = [(now, n_f, prev, m_f, m_u, n_un) for now in (False, True) for n_f in (0, 1, 50, 51) for prev in (0, 50)
            for m_f in (0, 10, 1000) for m_u in (0, 400, 40000) for n_un in (0, 1200, 1224, 1300)]
    rows += [(bool(rng.integers(2)), *map(int, rng.integers(0, 1 << 40, 5))) for _ in range(500)]
    return rows


@pytest.mark.parametrize("knobs", [{}, {"CUGRAPH_B200_BFS_ALPHA": "2.5", "CUGRAPH_B200_BFS_BETA": "0.75"}],
                         ids=["default", "set"])
def test_bfs_bottom_up_rule_emulated(surface, monkeypatch, knobs):
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    ref.set_knobs(monkeypatch, knobs)
    alpha = float(knobs.get("CUGRAPH_B200_BFS_ALPHA", 40.0))
    beta = float(knobs.get("CUGRAPH_B200_BFS_BETA", 24.0))
    L = _capi.lib()
    h = ResourceHandle(stream=0)
    for row in _bottom_up_table():
        now = row[0]
        got = L.cugraph_b200_bfs_bottom_up(h.ptr, int(now), *row[1:])
        assert got in (0, 1)
        assert bool(got) == ref.bottom_up_reference(alpha, beta, *row), row
    assert L.cugraph_b200_bfs_bottom_up(None, 1, 0, 0, 0, 0, 0) == 1      # no handle: the direction stays
    assert L.cugraph_b200_bfs_bottom_up(None, 0, 5, 0, 5, 0, 9) == 0


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_worker(rank, world, s, d, sources):
    """every schedule on this rank: the knobs are set before each graph's handle is made"""
    import torch
    from cugraph_b200 import mg
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    out = {}
    for name, (do, knobs) in ref.SCHEDULES.items():
        for k in ref.KNOBS:
            os.environ.pop(k, None)
        os.environ.update(knobs)
        g = mg.MGGraph(torch.from_numpy(s[lo:hi]), torch.from_numpy(d[lo:hi]))
        v, dist, pred = mg.bfs(g, torch.from_numpy(sources[rank]), direction_optimizing=do)
        again = mg.bfs(g, torch.from_numpy(sources[rank]), direction_optimizing=do)[2]
        out[name] = dict(v=v.numpy(), dist=dist.numpy(), pred=pred.numpy(), again=again.numpy(), stats=g.last_bfs_stats)
    return out


@pytest.mark.parametrize("world", [2, 4])
def test_mg_bfs_direction_emulated_gloo(world):
    rng = np.random.default_rng(world)
    s, d = refs.rmat_graph(8)
    for sym in (False, True):
        gs, gd = (np.concatenate([s, d]), np.concatenate([d, s])) if sym else (s, d)
        srcs = rng.choice(np.flatnonzero(np.bincount(gs) > 0), 3, replace=False).astype(np.int32)
        out = mg_procs.run(_gloo_worker, world, gs, gd, refs.split(srcs, world, rng), emulated=True)
        for name in ref.SCHEDULES:
            res = [o[name] for o in out]
            refs.check_bfs(gs, gd, res, srcs)
            assert all(np.array_equal(r["again"], r["pred"]) for r in res)
            st = res[0]["stats"]
            assert all(r["stats"] == st for r in res)
            assert (name != "top_down" or st["bottom_up"] == 0) and (name != "bottom_up" or st["top_down"] == 0), (name, st)
