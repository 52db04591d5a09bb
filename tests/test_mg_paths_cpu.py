"""Multi-GPU BFS from a set of sources and multi-GPU extract_paths on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running MGGraph.bfs and MGGraph.extract_paths: grids 1x2, 2x1,
  2x2 and 4x2 on a directed RMAT-8 and on a forest with forced predecessors.  Sources all from rank 0, split over the
  ranks, duplicated across ranks, all from a rank that owns none of them, with a depth limit, and none at all; distances
  bit-exact against the oracle, predecessors by the reference's predicate, paths against a numpy restatement of single
  GPU's walk, and on the forced forest bit-identical to single-GPU cugraph_extract_paths.
- cugraph_b200_paths_answer and cugraph_b200_paths_advance called directly against numpy, with empty batches and their
  error paths.
- World sizes 2, 4 and 8 over gloo with scattered 64-bit external ids (the real process groups)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_paths_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]


def _source_modes(sources, world, rng):
    """the sources given four ways: all from rank 0, split over the ranks, every id from two ranks, all from a rank that
    owns none of them"""
    empty = np.zeros(0, np.int32)
    src = np.asarray(sources, np.int32)
    free = world - 1
    assert not (refs.owned_by(src, world) == free).any()
    dup = [src[(np.arange(src.size) + r) % world < 2] for r in range(world)]
    return {"rank0": [src] + [empty] * (world - 1),
            "split": refs.split(src, world, rng),
            "duplicated": dup,
            "non_owner": [src if r == free else empty for r in range(world)]}


def _dests(s, d, world, rng, extra=()):
    """destinations for every rank: random vertices, ids that are not vertices, the extra ids; the last rank gets none"""
    ids = np.unique(np.concatenate([s, d]))
    pool = np.concatenate([rng.choice(ids, 60), refs.not_vertices(s, d), np.asarray(extra, np.int32)]).astype(np.int32)
    rng.shuffle(pool)
    parts = refs.split(pool, world - 1, rng) if world > 1 else [pool]
    return parts + [np.zeros(0, np.int32)] if world > 1 else parts


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_bfs_sources_and_paths_emulated(surface, monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    rng = np.random.default_rng(R * 10 + Cc)
    s, d = refs.rmat_graph(8)
    deg = np.bincount(s)
    cand = np.flatnonzero(deg > 0)
    cand = cand[refs.owned_by(cand, world) != world - 1]          # the last rank owns none of the sources
    srcs = rng.choice(cand, 4, replace=False).astype(np.int32)
    for mode, sources in _source_modes(srcs, world, rng).items():
        dests = _dests(s, d, world, rng, extra=srcs[:2])
        res = refs.mg_bfs_paths(s, d, world, sources, dests)
        refs.check_bfs(s, d, res, srcs)
        paths, length = refs.check_paths(res, dests)
        assert length > 1, mode
    # a depth limit
    dests = _dests(s, d, world, rng, extra=srcs)
    res = refs.mg_bfs_paths(s, d, world, refs.split(srcs, world, rng), dests, depth_limit=2)
    got_d = refs.check_bfs(s, d, res, srcs, depth_limit=2)
    assert got_d.max() == refs.IMAX and got_d[got_d < refs.IMAX].max() == 2
    refs.check_paths(res, dests)
    # no source on any rank: single GPU's result for an empty list, and paths of -1 of length 1
    res = refs.mg_bfs_paths(s, d, world, [np.zeros(0, np.int32)] * world, dests)
    for r in res:
        assert (r["dist"] == refs.IMAX).all() and (r["pred"] == -1).all()
        assert r["length"] == 1 and (r["paths"] == -1).all()
    refs.check_bfs(s, d, res, np.zeros(0, np.int32))


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_paths_forced_predecessors_emulated(surface, monkeypatch, R, Cc):
    """a forest in which every reached vertex has one in-neighbour one level closer: rows bit-identical to single GPU"""
    world = mg_world.grid_world(monkeypatch, R, Cc)
    rng = np.random.default_rng(5)
    s, d, roots, unreached = refs.forced_graph()
    ids = np.unique(np.concatenate([s, d]))
    pool = np.concatenate([ids, unreached[:5], roots, refs.not_vertices(s, d)]).astype(np.int32)
    rng.shuffle(pool)
    dests = refs.split(pool, world, rng)
    res = refs.mg_bfs_paths(s, d, world, refs.split(roots, world, rng), dests, repeat=True)
    refs.check_bfs(s, d, res, roots)
    paths, length = refs.check_paths(res, dests)
    sg_dist, sg_paths = refs.single_gpu_paths(s, d, roots, pool)
    assert np.array_equal(np.concatenate([r["paths"] for r in res]), sg_paths)
    assert length == sg_paths.shape[1]
    # every row: root ... destination along tree edges; unreached ids and non-vertices give rows of -1
    keys = set(zip(s.tolist(), d.tolist()))
    for row, t in zip(paths, pool.tolist()):
        if t >= sg_dist.size or sg_dist[t] < 0 or sg_dist[t] == refs.IMAX:
            assert (row == -1).all()
            continue
        k = int(sg_dist[t])
        assert row[k] == t and row[0] in set(roots.tolist()) and (row[k + 1:] == -1).all()
        assert all((int(a), int(b)) in keys for a, b in zip(row[:k], row[1:k + 1]))


def _bfs_forms_worker(rank, world, s, d, src):
    import torch
    g = mg_world.graph(rank, world, s, d)
    a = g.bfs(src)
    b = g.bfs(torch.tensor([src], dtype=torch.int32))
    c = g.bfs(np.int32(src), 3, False)
    return [x.numpy() for x in a], [x.numpy() for x in b], c[2]


def test_mg_bfs_scalar_and_one_element_forms_emulated(surface, monkeypatch):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d = refs.rmat_graph(8)
    for a, b, c in mg_world.run(world, _bfs_forms_worker, s, d, int(s[3])):
        for x, y in zip(a, b):
            assert x.dtype == y.dtype and np.array_equal(x, y)
        assert c is None


def _errors_worker(rank, world, s, d):
    import torch
    g = mg_world.graph(rank, world, s, d)
    good = torch.as_tensor(s[:2])
    out = {}
    out["invalid"] = refs._errors(g.bfs, torch.tensor([1 << 20] if rank == 1 else [], dtype=torch.int32))
    out["dtype"] = refs._errors(g.bfs, good.long() if rank == 0 else good)
    out["scalar"] = refs._errors(g.bfs, 1 << 20)
    v, dist, pred = g.bfs(good)
    dst = torch.as_tensor(d[:5])
    out["size"] = refs._errors(g.extract_paths, dist[:-1] if rank == 2 else dist, pred, dst)
    out["none"] = refs._errors(g.extract_paths, dist, None if rank == 3 else pred, dst)
    out["dist_dtype"] = refs._errors(g.extract_paths, dist.long() if rank == 1 else dist, pred, dst)
    paths, length = g.extract_paths(dist, pred, dst)      # the graph still works after the errors
    out["ok"] = (paths.shape[0], length)
    return out


def test_mg_bfs_and_paths_errors_on_every_rank_emulated(surface, monkeypatch):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d = refs.rmat_graph(8)
    res = mg_world.run(world, _errors_worker, s, d)
    want = {"invalid": "CugraphValueError", "dtype": "TypeError", "scalar": "ValueError", "size": "ValueError",
            "none": "ValueError", "dist_dtype": "TypeError"}
    for key, name in want.items():
        got = [r[key] for r in res]
        assert all(g == got[0] for g in got), (key, got)
        assert got[0][0] == name, (key, got[0])
    assert "Found invalid vertex in the input sources" in res[0]["invalid"][1]
    assert all(r["ok"][0] == 5 for r in res)


# ---------------------------------------------------------------------------------------------------- the entry points
def _call(name, *tensors_and_scalars):
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    import torch
    L = _capi.lib()
    handle = ResourceHandle(stream=0)
    views, args = [], []
    for x in tensors_and_scalars:
        if isinstance(x, torch.Tensor):
            views.append(View(x))
            args.append(views[-1].ptr)
        else:
            args.append(x)
    err = C.c_void_p()
    try:
        code = getattr(L, name)(handle.ptr, *args, C.byref(err))
        _capi.check(code, err, name)
    finally:
        for v in views:
            v.free()


def test_paths_answer_against_numpy_emulated(surface):
    import torch
    rng = np.random.default_rng(1)
    n_local = 500
    codes = rng.integers(-1, 1 << 40, n_local)
    for vdt in (torch.int32, torch.int64):
        verts = torch.as_tensor(rng.permutation(10**6)[:n_local]).to(vdt)
        lids = rng.integers(-3, n_local + 3, 2000).astype(np.int32)
        ans = torch.full((2 * lids.size,), 7, dtype=torch.int64)
        _call("cugraph_b200_paths_answer", torch.as_tensor(lids), verts, torch.as_tensor(codes), n_local, ans)
        ok = (lids >= 0) & (lids < n_local)
        li = np.where(ok, lids, 0)
        a = ans.numpy().reshape(-1, 2)
        assert np.array_equal(a[:, 0], np.where(ok, verts.numpy().astype(np.int64)[li], -1))
        assert np.array_equal(a[:, 1], np.where(ok, codes[li], -1))
        empty = torch.zeros(0, dtype=torch.int32)
        _call("cugraph_b200_paths_answer", empty, verts, torch.as_tensor(codes), n_local, torch.zeros(0, dtype=torch.int64))


def _advance(ans, rows, pos, paths, length, maxpart, world, cap):
    import torch
    nxt = [torch.full((cap,), -9, dtype=torch.int32) for _ in range(3)]
    counts = torch.full((world,), -9, dtype=torch.int64)
    _call("cugraph_b200_paths_advance", ans, rows, pos, paths.view(-1), length, maxpart, world, *nxt, counts)
    return [x.numpy() for x in nxt], counts.numpy()


def test_paths_advance_against_numpy_emulated(surface):
    import torch
    rng = np.random.default_rng(2)
    world, maxpart, n_rows, length, n = 5, 300, 400, 9, 3000
    rows = rng.integers(-2, n_rows + 2, n).astype(np.int32)
    pos = rng.integers(-1, length + 1, n).astype(np.int32)
    ext = rng.integers(0, 1 << 31, n)
    code = np.where(rng.random(n) < 0.2, -1, rng.integers(0, (world + 1) * maxpart, n))   # some name no rank
    ans = torch.as_tensor(np.stack([ext, code], 1).reshape(-1))
    inside = (rows >= 0) & (rows < n_rows) & (pos >= 0) & (pos < length)
    q = code // maxpart
    goes = inside & (pos > 0) & (code >= 0) & (q < world)
    for vdt in (torch.int32, torch.int64):
        paths = torch.full((n_rows, length), -1, dtype=vdt)
        (nl, nr, npos), counts = _advance(ans, torch.as_tensor(rows), torch.as_tensor(pos), paths, length, maxpart, world, n)
        idx = np.flatnonzero(inside)
        assert np.array_equal(np.bincount(q[goes], minlength=world), counts)
        at = 0
        for r in range(world):
            sel = goes & (q == r)
            got = sorted(zip(nl[at:at + counts[r]].tolist(), nr[at:at + counts[r]].tolist(), npos[at:at + counts[r]].tolist()))
            exp = sorted(zip((code[sel] - r * maxpart).tolist(), rows[sel].tolist(), (pos[sel] - 1).tolist()))
            assert got == exp, r
            at += counts[r]
        assert (nl[at:] == -9).all()
        # the matrix: every (row, pos) of an entry inside it holds that entry's id (one of them where entries share it)
        p = paths.numpy().astype(np.int64)
        wrote = np.zeros((n_rows, length), bool)
        wrote[rows[idx], pos[idx]] = True
        assert (p[~wrote] == -1).all()
        cand = {}
        for i in idx.tolist():
            cand.setdefault((int(rows[i]), int(pos[i])), set()).add(int(ext[i]))
        assert all(int(p[k]) in v for k, v in cand.items())
    # an empty batch: counts zeroed, nothing written
    paths = torch.full((3, 4), -1, dtype=torch.int32)
    e32, e64 = torch.zeros(0, dtype=torch.int32), torch.zeros(0, dtype=torch.int64)
    _, counts = _advance(e64, e32, e32, paths, 4, 10, 3, 1)
    assert (counts == 0).all() and (paths.numpy() == -1).all()


def test_paths_entry_errors_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    i32, i64 = torch.int32, torch.int64
    lids, verts, codes, ans = torch.zeros(4, dtype=i32), torch.zeros(6, dtype=i32), torch.zeros(6, dtype=i64), torch.zeros(8, dtype=i64)
    base = dict(lids=lids, verts=verts, codes=codes, n_local=6, ans=ans)
    for kw in (dict(lids=lids.long()), dict(verts=verts.float()), dict(codes=codes.int()), dict(ans=ans.int()),
               dict(ans=ans[:7]), dict(n_local=7), dict(verts=verts[:5])):
        a = dict(base, **kw)
        with pytest.raises(_capi.CugraphError) as e:
            _call("cugraph_b200_paths_answer", a["lids"], a["verts"], a["codes"], a["n_local"], a["ans"])
        assert e.value.code == _capi.INVALID_INPUT, kw
    rows, pos, paths = torch.zeros(4, dtype=i32), torch.zeros(4, dtype=i32), torch.zeros(12, dtype=i32)
    nxt, cnt = [torch.zeros(4, dtype=i32) for _ in range(3)], torch.zeros(3, dtype=i64)
    base = dict(ans=ans, rows=rows, pos=pos, paths=paths, length=3, maxpart=5, world=3, nl=nxt[0], nr=nxt[1], np_=nxt[2],
                counts=cnt)
    for kw in (dict(ans=ans[:7]), dict(ans=ans.int()), dict(rows=rows.long()), dict(pos=pos[:3]), dict(paths=paths.float()),
               dict(length=0), dict(length=5), dict(maxpart=0), dict(world=0), dict(nl=nxt[0][:3]), dict(nr=nxt[1].long()),
               dict(counts=cnt[:2]), dict(counts=cnt.int())):
        a = dict(base, **kw)
        with pytest.raises(_capi.CugraphError) as e:
            _call("cugraph_b200_paths_advance", a["ans"], a["rows"], a["pos"], a["paths"], a["length"], a["maxpart"],
                  a["world"], a["nl"], a["nr"], a["np_"], a["counts"])
        assert e.value.code == _capi.INVALID_INPUT, kw


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_graph():
    """the forced forest with scattered 64-bit external ids"""
    s, d, roots, unreached = refs.forced_graph(seed=9)
    ids = np.random.default_rng(9).choice(10**9, size=int(max(s.max(), d.max())) + 1, replace=False).astype(np.int64) + 10**10
    return ids, s, d, roots, unreached


def _gloo_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    ids, s, d, roots, unreached = _gloo_graph()
    rng = np.random.default_rng(world)
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    g = mg.MGGraph(torch.from_numpy(ids[s[lo:hi]]), torch.from_numpy(ids[d[lo:hi]]))
    src = refs.split(roots, world, rng)[rank]
    dests = refs.split(np.concatenate([np.unique(np.concatenate([s, d])), unreached[:3], roots]), world, rng)[rank]
    v, dist, pred = mg.bfs(g, torch.from_numpy(ids[src]))
    dst = torch.from_numpy(np.concatenate([ids[dests], [5, 7]]))     # two ids that are not vertices
    paths, length = mg.extract_paths(g, dist, pred, dst)
    return dict(v=v.numpy(), dist=dist.numpy(), pred=pred.numpy(), paths=paths.numpy(), length=length,
                rounds=g.last_paths_stats["rounds"], dests=dst.numpy())


@pytest.mark.parametrize("world", [2, 4, 8])
def test_mg_paths_emulated_gloo(world):
    res = mg_procs.run(_gloo_worker, world, emulated=True)
    ids, s, d, roots, _ = _gloo_graph()
    for r in res:
        assert r["v"].dtype == np.int64 and r["paths"].dtype == np.int64
    k_of = {int(x): k for k, x in enumerate(ids)}
    local = [dict(r, v=np.array([k_of[int(x)] for x in r["v"]], np.int32),
                  pred=np.array([k_of[int(x)] if x >= 0 else -1 for x in r["pred"]], np.int64)) for r in res]
    refs.check_bfs(s, d, local, roots)
    _, length = refs.check_paths(res, [r["dests"] for r in res])
    assert length > 2
