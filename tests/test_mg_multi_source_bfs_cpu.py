"""Multi-GPU multi-source BFS on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running MGGraph.multi_source_bfs: grids 1x2, 2x1, 2x2 and 4x2,
  the four schedules of tests/mg_bfs_direction_ref.py, its graphs (directed and symmetrised RMAT-8, a path with int64
  external ids, a grid with edges removed, a lollipop, small components, a forest), 1, 63, 64, 65 and 130 sources with a
  duplicate, depth limits 0, 1, 3 and none.  Every row: distances bit-exact against the oracle, predecessors by the
  largest-code rule; the first, 65th and last rows bit-identical to MGGraph.bfs from their source, valid by
  MGGraph.validate_bfs, and the same extract_paths; last_ms_bfs_stats' level counts.
- An isolated vertex given through vertices=, an edgeless graph, self-loops and multi-edges, no sources,
  compute_predecessors=False and a repeated call; every error, raised on every rank.
- The five entry points against numpy on one block, with their argument errors.
- World sizes 2 and 4 over gloo."""
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
from tests.emu_py import surface  # noqa: E402, F401
from tests.test_traversal_shapes_gpu import EMU_SIZES  # noqa: E402

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]
SIZES = dict(EMU_SIZES, path=30, grid=6, tail=12, components=30)   # every level is a round of collectives
LIMITS = (-1, 0, 1, 3)


@pytest.mark.parametrize("schedule", list(dref.SCHEDULES))
@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_multi_source_bfs_emulated(surface, monkeypatch, R, Cc, schedule):
    """each graph with a source count and a depth limit that rotate over the grids and schedules, so that every count
    and every limit meets every graph"""
    world = mg_world.grid_world(monkeypatch, R, Cc)
    dref.set_knobs(monkeypatch, dref.SCHEDULES[schedule][1])
    gi, si = GRIDS.index((R, Cc)), list(dref.SCHEDULES).index(schedule)
    rng = np.random.default_rng(gi * 10 + si)
    for i, case in enumerate(dref.cases(SIZES, 8)):
        n = ref.SOURCE_COUNTS[(i + gi + si) % len(ref.SOURCE_COUNTS)]
        limit = LIMITS[(i + 2 * gi + si) % len(LIMITS)]
        ref.run_case(case, world, schedule, n, limit, rng)


# ------------------------------------------------------------------------------------------------ inputs and errors
def _inputs_worker(rank, world, s, d, vertices, sources):
    import torch
    from cugraph_b200 import mg
    s_r, d_r = mg_world.share(rank, world, s, d)
    g = mg.MGGraph(torch.as_tensor(s_r), torch.as_tensor(d_r), vertices=torch.as_tensor(vertices))
    src = torch.as_tensor(sources)
    v, dist, pred = mg.multi_source_bfs(g, src)
    stats = dict(g.last_ms_bfs_stats)
    v2, dist2, pred2 = g.multi_source_bfs(src)
    _, dist3, none = g.multi_source_bfs(src, compute_predecessors=False)
    _, d0, p0 = g.multi_source_bfs(src[:0])
    return dict(v=v.numpy(), dist=dist.numpy(), pred=pred.numpy(), n_local=g.part.n_local, stats=stats,
                same=bool(torch.equal(v, v2) and torch.equal(dist, dist2) and torch.equal(pred, pred2)
                          and torch.equal(dist, dist3)) and none is None,
                empty=(tuple(d0.shape), tuple(p0.shape), p0.dtype == v.dtype), empty_stats=dict(g.last_ms_bfs_stats))


def test_mg_multi_source_bfs_inputs_emulated(surface, monkeypatch):
    """isolated vertices, an edgeless graph, self-loops and multi-edges; no sources; no predecessors; a repeated call"""
    world = mg_world.grid_world(monkeypatch, 2, 2)
    rng = np.random.default_rng(11)
    s, d = refs.rmat_graph(7)
    s = np.concatenate([s, [3, 3, 5], s[:40]]).astype(np.int32)      # self-loops and more multi-edges
    d = np.concatenate([d, [3, 3, 5], d[:40]]).astype(np.int32)
    iso = np.int32(int(max(s.max(), d.max())) + 4)
    for gs, gd, extra in ((s, d, [iso, iso + 2]), (np.zeros(0, np.int32), np.zeros(0, np.int32), [1, 4, 9])):
        verts = np.unique(np.concatenate([gs, gd, extra])).astype(np.int32)
        srcs = np.concatenate([rng.choice(verts, 70), [extra[0], extra[0]]]).astype(np.int32)
        res = mg_world.run(world, _inputs_worker, gs, gd, np.asarray(extra, np.int32), srcs)
        vids, dist, pred, _ = ref.gather(res)
        assert np.array_equal(np.sort(vids), verts)
        for r in res:
            assert r["same"] and r["empty"] == ((0, r["n_local"]), (0, r["n_local"]), True)
            assert r["empty_stats"] == dict(batches=0, levels=0, top_down=0, bottom_up=0)
            assert r["stats"]["batches"] == 2
        # the isolated source reaches itself only
        for k in (len(srcs) - 2, len(srcs) - 1):
            row = np.where(vids == extra[0], 0, refs.IMAX)
            assert np.array_equal(dist[k], row) and (pred[k] == -1).all()
        ref.check_rows(gs, gd, res, srcs, vertices=extra)


def _errors_worker(rank, world, s, d, bad):
    import torch
    g = mg_world.graph(rank, world, s, d)
    good = torch.as_tensor(np.asarray([s[0], d[1], s[2]], np.int32))
    cases = {"dtype": good.long() if rank == world - 1 else good,
             "not a vertex": torch.as_tensor(np.asarray([s[0], bad], np.int32)),
             "length": good[:2] if rank == 1 else good,
             "order": good.flip(0) if rank == 0 else good,
             "value": torch.where(torch.arange(3) == 1, torch.tensor(bad, dtype=torch.int32), good) if rank == world - 1
             else good}
    out = {}
    for name, src in cases.items():
        try:
            g.multi_source_bfs(src)
            out[name] = None
        except Exception as e:  # noqa: BLE001
            out[name] = (type(e).__name__, str(e))
    out["after"] = g.multi_source_bfs(good)[1].numpy().shape
    return out


def test_mg_multi_source_bfs_errors_emulated(surface, monkeypatch):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d = refs.rmat_graph(6)
    bad = int(refs.not_vertices(s, d, 1)[0])
    res = mg_world.run(world, _errors_worker, s, d, bad)
    want = {"dtype": ("TypeError", "dtype of the edge ids"), "not a vertex": ("CugraphValueError", "invalid vertex"),
            "length": ("ValueError", "same list"), "order": ("ValueError", "same list"), "value": ("ValueError", "same list")}
    for r in res:
        for name, (cls, text) in want.items():
            assert r[name] is not None and r[name][0] == cls and text in r[name][1], (name, r[name])
        assert r["after"][0] == 3


# ---------------------------------------------------------------------------------------------------- the entry points
def _block(rng, n_rows, n_cols, m):
    rows = rng.integers(0, n_rows, m).astype(np.int32)
    cols = rng.integers(0, n_cols, m).astype(np.int32)
    rows[: m // 8] = 3          # a dense row: the warp kernels
    cols[m // 8: m // 4] = 5    # a hub column: the merge-path advance splits its edges
    return rows, cols, dref.Block(rows, cols, n_rows, n_cols)


def _words(rng, n, p, nb):
    """n random words of nb bits, each bit set with probability p"""
    bits = rng.random((n, nb)) < p
    return (bits.astype(np.uint64) << np.arange(nb, dtype=np.uint64)).sum(1, dtype=np.uint64).view(np.int64)


def check_block_steps(b, rows, cols, n_rows, n_cols, rng, device, trials):
    import torch
    t = lambda a: torch.as_tensor(a).to(device)  # noqa: E731
    for maxpart, grid_cols, grid_c, nb, pc, ps in trials:
        cur = _words(rng, n_cols, pc, nb)
        seen = _words(rng, n_rows, ps, nb)
        want = ref.step_reference(rows, cols, n_rows, cur, seen, nb)
        for fn in ("cugraph_b200_block_ms_bfs_push", "cugraph_b200_block_ms_bfs_pull"):
            nxt = torch.full((n_rows + 3,), 77, dtype=torch.int64, device=device)    # stale values and a longer array
            b.call(fn, t(cur), t(seen), nb, nxt)
            got = nxt.cpu().numpy()
            assert np.array_equal(got[:n_rows], want), fn
            assert (got[n_rows:] == 77).all(), fn
        # predecessors of the rows that gained bits, with the segments sized from the new bits
        new = want
        pc_rows = np.array([bin(int(x) & (2**64 - 1)).count("1") for x in new], np.int64)
        seg_lens = [pc_rows[k * maxpart:(k + 1) * maxpart].sum() for k in range(grid_cols)]
        for seg in sorted({int(max(seg_lens)), int(max(seg_lens)) + 5, max(int(max(seg_lens)) // 2, 1)}):
            pairs = torch.full((grid_cols * seg + 2,), 77, dtype=torch.int64, device=device)
            b.call("cugraph_b200_block_ms_bfs_pred", t(cur), t(new), maxpart, grid_cols, grid_c, seg, pairs)
            got = pairs.cpu().numpy()
            assert np.array_equal(got[:grid_cols * seg], ref.pred_reference(rows, cols, n_rows, cur, new, maxpart, grid_cols,
                                                                             grid_c, seg)), seg
            assert (got[grid_cols * seg:] == 77).all()


def test_block_ms_bfs_steps_against_numpy_emulated(surface):
    rng = np.random.default_rng(4)
    n_rows, n_cols = 600, 900
    rows, cols, b = _block(rng, n_rows, n_cols, 5000)
    try:
        check_block_steps(b, rows, cols, n_rows, n_cols, rng, "cpu",
                          ((300, 2, 1, 64, 0.05, 0.3), (200, 3, 0, 7, 0.5, 0.0), (600, 1, 0, 1, 0.0, 0.5),
                           (150, 4, 3, 40, 0.9, 0.9)))
    finally:
        b.close()


def check_owner_steps(rng, device, trials):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    import ctypes as C
    L = _capi.lib()
    h = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream if device != "cpu" else 0)

    def call(name, *args):
        views, a = [], []
        for x in args:
            if isinstance(x, torch.Tensor) or x is None:
                views.append(View(x))
                a.append(views[-1].ptr)
            else:
                a.append(x)
        err = C.c_void_p()
        try:
            _capi.check(getattr(L, name)(h.ptr, *a, C.byref(err)), err, name)
        finally:
            for v in views:
                v.free()

    t = lambda a: torch.tensor(np.ascontiguousarray(a)).to(device)  # a copy: the calls update some arrays in place  # noqa: E731
    for parts, maxpart, n_local, nb, level, with_deg in trials:
        recv = np.concatenate([_words(rng, maxpart, 0.1, nb) for _ in range(parts)])
        seen = _words(rng, maxpart, 0.4, nb)
        seen[: n_local // 5] = -1 if nb == 64 else (1 << nb) - 1 - 1     # nearly whole words: some become whole
        cur = _words(rng, maxpart, 0.3, nb)
        dist = rng.integers(0, 5, nb * n_local).astype(np.int32)
        dout = rng.integers(0, 100, n_local).astype(np.int64) if with_deg else None
        din = rng.integers(0, 100, n_local).astype(np.int64) if with_deg else None
        ts, tc, td, tk = t(seen), t(cur), t(dist), torch.full((6,), 9, dtype=torch.int64, device=device)
        call("cugraph_b200_ms_bfs_owner_step", t(recv), parts, maxpart, n_local, nb, level, ts, tc, td,
             None if dout is None else t(dout), None if din is None else t(din), tk)
        w_seen, w_cur, w_dist, w_counts = ref.owner_step_reference(recv, parts, maxpart, n_local, nb, level, seen, cur, dist,
                                                                   dout, din)
        assert np.array_equal(ts.cpu().numpy(), w_seen) and np.array_equal(tc.cpu().numpy(), w_cur)
        assert np.array_equal(td.cpu().numpy(), w_dist)
        assert np.array_equal(tk.cpu().numpy()[:5], w_counts) and tk.cpu().numpy()[5] == 9
        # the scatter of the owner's pairs into the predecessor rows (also with a short pair buffer)
        n_bits = int(w_counts[4])
        for n_pairs in (n_bits, n_bits // 2):
            pairs = rng.integers(0, 1 << 40, n_pairs).astype(np.int64)
            pred = rng.integers(-1, 3, nb * n_local).astype(np.int64)
            tp = t(pred)
            call("cugraph_b200_ms_bfs_owner_pred", tc, t(pairs), n_local, nb, tp)
            assert np.array_equal(tp.cpu().numpy(), ref.owner_pred_reference(w_cur, pairs, n_local, nb, pred))


def test_ms_bfs_owner_steps_against_numpy_emulated(surface):
    check_owner_steps(np.random.default_rng(8), "cpu", ((1, 300, 300, 64, 3, True), (3, 200, 150, 5, 1, False),
                                                        (4, 100, 0, 1, 2, True), (2, 500, 480, 33, 7, True)))


def test_ms_bfs_entry_point_errors_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    rng = np.random.default_rng(5)
    n_rows, n_cols = 40, 60
    _, _, b = _block(rng, n_rows, n_cols, 300)
    i64 = torch.int64
    cur, seen, nxt = torch.zeros(n_cols, dtype=i64), torch.zeros(n_rows, dtype=i64), torch.zeros(n_rows, dtype=i64)
    steps = {"cur dtype": (cur.int(), seen, 3, nxt), "seen dtype": (cur, seen.double(), 3, nxt),
             "next dtype": (cur, seen, 3, nxt.int()), "short cur": (cur[:-1], seen, 3, nxt),
             "short seen": (cur, seen[:-1], 3, nxt), "short next": (cur, seen, 3, nxt[:-1]), "zero sources": (cur, seen, 0, nxt),
             "65 sources": (cur, seen, 65, nxt)}
    want = {"cur dtype": "must be INT64", "seen dtype": "must be INT64", "next dtype": "must be INT64",
            "short cur": "shorter", "short seen": "shorter", "short next": "shorter", "zero sources": "n_sources",
            "65 sources": "n_sources"}
    pairs = torch.zeros(100, dtype=i64)
    preds = {"cur dtype": (cur.int(), nxt, 20, 2, 1, 10, pairs), "pairs dtype": (cur, nxt, 20, 2, 1, 10, pairs.int()),
             "short new": (cur, nxt[:-1], 20, 2, 1, 10, pairs), "short pairs": (cur, nxt, 20, 2, 1, 51, pairs),
             "grid_c": (cur, nxt, 20, 2, 2, 10, pairs), "maxpart": (cur, nxt, 0, 2, 0, 10, pairs),
             "rows past the grid": (cur, nxt, 10, 2, 0, 10, pairs)}
    want_pred = {"cur dtype": "must be INT64", "pairs dtype": "must be INT64", "short new": "shorter",
                 "short pairs": "grid_cols * seg", "grid_c": "bad grid position", "maxpart": "bad grid position",
                 "rows past the grid": "more row slots"}
    try:
        for name, args in steps.items():
            for fn in ("cugraph_b200_block_ms_bfs_push", "cugraph_b200_block_ms_bfs_pull"):   # the same checks
                with pytest.raises(_capi.CugraphError) as e:
                    b.call(fn, *args)
                assert e.value.code == _capi.INVALID_INPUT and want[name] in str(e.value), (fn, name, str(e.value))
        for name, args in preds.items():
            with pytest.raises(_capi.CugraphError) as e:
                b.call("cugraph_b200_block_ms_bfs_pred", *args)
            assert e.value.code == _capi.INVALID_INPUT and want_pred[name] in str(e.value), (name, str(e.value))
        b.call("cugraph_b200_block_ms_bfs_push", cur, seen, 3, nxt)    # the block still works
        assert (nxt.numpy() == 0).all()
    finally:
        b.close()
    _owner_errors()


def _owner_errors():
    import ctypes as C
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    h = ResourceHandle(stream=0)
    i64 = torch.int64
    z = lambda n, dt=i64: torch.zeros(n, dtype=dt)  # noqa: E731
    base = dict(recv=z(20), parts=2, maxpart=10, n_local=8, nb=3, level=1, seen=z(8), cur=z(8), dist=z(24, torch.int32),
                dout=None, din=None, counts=z(5))
    cases = {"recv dtype": dict(recv=z(20, torch.int32)), "short recv": dict(recv=z(19)), "dist dtype": dict(dist=z(24)),
             "short dist": dict(dist=z(23, torch.int32)), "short seen": dict(seen=z(7)), "short counts": dict(counts=z(4)),
             "one degree": dict(dout=z(8)), "degree dtype": dict(dout=z(8, torch.int32), din=z(8, torch.int32)),
             "n_local": dict(n_local=11), "level": dict(level=0), "parts": dict(parts=0), "sources": dict(nb=65)}
    want = {"recv dtype": "must be INT64", "short recv": "parts * maxpart", "dist dtype": "INT32", "short dist": "n_sources",
            "short seen": "shorter than n_local", "short counts": "5 entries", "one degree": "both degree arrays",
            "degree dtype": "degrees must be INT64", "n_local": "bad parts", "level": "bad parts", "parts": "bad parts",
            "sources": "n_sources"}

    def call(name, *args):
        views, a = [], []
        for x in args:
            if isinstance(x, torch.Tensor) or x is None:
                views.append(View(x))
                a.append(views[-1].ptr)
            else:
                a.append(x)
        err = C.c_void_p()
        try:
            _capi.check(getattr(L, name)(h.ptr, *a, C.byref(err)), err, name)
        finally:
            for v in views:
                v.free()

    for name, kw in cases.items():
        a = dict(base, **kw)
        with pytest.raises(_capi.CugraphError) as e:
            call("cugraph_b200_ms_bfs_owner_step", a["recv"], a["parts"], a["maxpart"], a["n_local"], a["nb"], a["level"],
                 a["seen"], a["cur"], a["dist"], a["dout"], a["din"], a["counts"])
        assert e.value.code == _capi.INVALID_INPUT and want[name] in str(e.value), (name, str(e.value))
    for args, text in (((z(7), z(4), 8, 3, z(24)), "shorter than n_local"), ((z(8), z(4, torch.int32), 8, 3, z(24)), "INT64"),
                       ((z(8), z(4), 8, 3, z(23)), "n_sources * n_local"), ((z(8), z(4), 8, 0, z(24)), "n_sources")):
        with pytest.raises(_capi.CugraphError) as e:
            call("cugraph_b200_ms_bfs_owner_pred", *args)
        assert e.value.code == _capi.INVALID_INPUT and text in str(e.value), (text, str(e.value))


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_worker(rank, world, s, d, sources):
    import torch
    from cugraph_b200 import mg
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    out = {}
    for name, (do, knobs) in dref.SCHEDULES.items():
        for k in dref.KNOBS:
            os.environ.pop(k, None)
        os.environ.update(knobs)
        g = mg.MGGraph(torch.from_numpy(s[lo:hi]), torch.from_numpy(d[lo:hi]))
        v, dist, pred = mg.multi_source_bfs(g, torch.from_numpy(sources), direction_optimizing=do)
        _, d1, p1 = g.bfs(int(sources[-1]))
        same = torch.equal(dist[-1], d1) and torch.equal(pred[-1], p1)
        out[name] = dict(v=v.numpy(), dist=dist.numpy(), pred=pred.numpy(), n_local=g.part.n_local,
                         stats=g.last_ms_bfs_stats, same=same)
    return out


@pytest.mark.parametrize("world", [2, 4])
def test_mg_multi_source_bfs_emulated_gloo(world):
    rng = np.random.default_rng(world)
    s, d = refs.rmat_graph(7)
    for gs, gd in ((s, d), (np.concatenate([s, d]), np.concatenate([d, s]))):
        srcs = rng.choice(np.unique(np.concatenate([gs, gd])), 66).astype(np.int32)
        out = mg_procs.run(_gloo_worker, world, gs, gd, srcs, emulated=True)
        for name in dref.SCHEDULES:
            res = [o[name] for o in out]
            ecc = ref.check_rows(gs, gd, res, srcs)
            st = res[0]["stats"]
            assert all(r["stats"] == st and r["same"] for r in res), name
            assert st["levels"] == ref.expected_levels(ecc, -1) and st["batches"] == 2, (name, st)
