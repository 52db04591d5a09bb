"""Multi-source BFS (cugraph_b200_multi_source_bfs through cugraph_b200.traversal.multi_source_bfs and api.multi_source_bfs)
on the GPU.

Row s of a result is checked against cugraph_bfs from the single source sources[s] with the same depth limit: the same
vertices order, the same dtype and bit-equal distances.  On small graphs every row is also checked against the CPU oracle's
BFS.  Predecessors are checked row by row with the reference tests' validity predicate (oracle.check_bfs_predecessors,
restated over all rows at once in _assert_pred_rows): -1 for the source and the unreached vertices, else an in-neighbour one
level closer.  Batches hold 64 sources, so 63 / 64 / 65 / 130 sources cover both sides of the batch boundary.

The check_* functions are shared with tests/test_multi_source_bfs_cpu.py, which runs them on the CPU emulation of the
library at smaller sizes."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle.rmat import rmat_edgelist
from tests.gpu_util import make_graph
from tests.test_paths_gpu import BFS_SCHEDULES, OFFS64

pytestmark = pytest.mark.gpu

INT_MAX = 2**31 - 1
N_SOURCES = (1, 5, 63, 64, 65, 130)
LIMITS = (0, 1, 3)  # 0: no depth limit


def _graph(monkeypatch, knobs, *args, **kw):
    """make_graph with CUGRAPH_B200_<knob> set while its handle is created (the handle reads the knobs once)"""
    for k, v in knobs.items():
        monkeypatch.setenv("CUGRAPH_B200_" + k, v)
    try:
        return make_graph(*args, **kw)
    finally:
        for k in knobs:
            monkeypatch.delenv("CUGRAPH_B200_" + k)


def edges(kind, size, seed):
    """(src, dst, V, symmetric): 'random' (V = size, 4 V directed edges), 'rmat' (scale = size, edge factor 16), each
    directed or, with the suffix '_sym', with every edge in both directions"""
    base = kind.removesuffix("_sym")
    if base == "random":
        V = size
        rng = np.random.default_rng(seed)
        s, d = rng.integers(0, V, 4 * V).astype(np.int32), rng.integers(0, V, 4 * V).astype(np.int32)
    else:
        s, d = rmat_edgelist(size, 16 << size, seed=seed)
        s, d, V = np.asarray(s, np.int32), np.asarray(d, np.int32), 1 << size
    sym = kind.endswith("_sym")
    if sym:
        s, d = np.concatenate([s, d]), np.concatenate([d, s])
    return s, d, V, sym


def ms_bfs(h, g, sources, depth_limit=0, compute_predecessors=True, vertex_dtype=np.int32):
    """(distances [n, V], predecessors [n, V] or None, vertices [V]) as numpy arrays"""
    import torch
    from cugraph_b200.traversal import multi_source_bfs
    dist, pred, verts = multi_source_bfs(h, g, torch.as_tensor(np.asarray(sources, vertex_dtype)).cuda(), depth_limit,
                                         compute_predecessors)
    return dist.cpu().numpy(), None if pred is None else pred.cpu().numpy(), verts.cpu().numpy()


def single_bfs(h, g, source, depth_limit=0, vertex_dtype=np.int32):
    """cugraph_bfs from one source, top-down: (distances, predecessors, vertices) as numpy arrays"""
    import torch
    from cugraph_b200 import pylibcugraph as plc
    dist, pred, verts = plc.bfs(h, g, torch.as_tensor(np.asarray([source], vertex_dtype)).cuda(), False, depth_limit, True, False)
    return dist.cpu().numpy(), pred.cpu().numpy(), verts.cpu().numpy()


def _by_id(verts, rows):
    """columns of rows [n, V] in reported order -> indexed by external id (the ids are 0 .. V-1)"""
    out = np.empty_like(rows)
    out[:, verts] = rows
    return out


def _assert_pred_rows(s, d, V, sources, dist, pred):
    """oracle.check_bfs_predecessors for every row at once; dist / pred indexed by external id"""
    inf = np.iinfo(dist.dtype).max
    keys = np.unique(np.asarray(s, np.int64) * V + np.asarray(d, np.int64))
    rows = np.arange(len(sources))
    reached = dist != inf
    assert (pred[~reached] == -1).all(), "an unreached vertex has a predecessor"
    assert (pred[rows, np.asarray(sources, np.int64)] == -1).all(), "a source has a predecessor"
    is_src = np.zeros(dist.shape, bool)
    is_src[rows, np.asarray(sources, np.int64)] = True
    r, v = np.nonzero(reached & ~is_src)
    p = pred[r, v].astype(np.int64)
    assert (p >= 0).all(), "a reached vertex has no predecessor"
    assert (dist[r, p].astype(np.int64) + 1 == dist[r, v].astype(np.int64)).all(), "a predecessor is not one level closer"
    q = p * V + v
    pos = np.minimum(np.searchsorted(keys, q), max(keys.size - 1, 0))
    assert q.size == 0 or (keys[pos] == q).all(), "a predecessor is not an in-neighbour"


def _pick_sources(s, V, n, seed):
    """n distinct vertices: the largest out-degree hub, an isolated vertex if there is one, the rest at random"""
    deg = np.bincount(s, minlength=V)
    rng = np.random.default_rng(seed)
    first = [int(deg.argmax())] + [int(x) for x in np.flatnonzero(deg == 0)[:1]]
    rest = rng.permutation(np.setdiff1d(np.arange(V), first))[: n - len(first)]
    return np.concatenate([first, rest]).astype(np.int64)[:n]


def check_rows(monkeypatch, kind, size, n_sources=N_SOURCES, limits=LIMITS, knobs=None, seed=0, with_oracle=False, **kw):
    """row parity with cugraph_bfs for every n in n_sources and every depth limit (and with the CPU oracle), predecessors
    valid; kw: store_transposed, renumber, vertex_dtype"""
    s, d, V, sym = edges(kind, size, seed)
    vdt = kw.get("vertex_dtype", np.int32)
    h, g = _graph(monkeypatch, knobs or {}, s, d, symmetric=sym, vertices=np.arange(V, dtype=vdt), **kw)
    srcs_all = _pick_sources(s, V, max(n_sources), seed)
    csr = oracle.coo_to_csx(s, d, V) if with_oracle else None
    ref = {}
    for limit in limits:
        for n in n_sources:
            srcs = srcs_all[:n]
            dist, pred, verts = ms_bfs(h, g, srcs, limit, vertex_dtype=vdt)
            assert dist.shape == (n, V) and pred.shape == (n, V) and dist.dtype == vdt and pred.dtype == vdt
            for k, src in enumerate(srcs.tolist()):
                if (src, limit) not in ref:
                    rd, _, rv = single_bfs(h, g, src, limit, vdt)
                    ref[(src, limit)] = (rd, rv)
                rd, rv = ref[(src, limit)]
                case = f"{kind}/{size} {kw} n_sources={n} row {k} (source {src}) depth_limit={limit}"
                assert np.array_equal(verts, rv), case
                assert dist[k].dtype == rd.dtype and np.array_equal(dist[k], rd), case
            dist_id, pred_id = _by_id(verts, dist), _by_id(verts, pred)
            _assert_pred_rows(s, d, V, srcs, dist_id, pred_id)
            if with_oracle:
                for k, src in enumerate(srcs.tolist()):
                    od, _ = oracle.bfs(s, d, V, [src], depth_limit=limit or None, csr=csr)
                    assert np.array_equal(dist_id[k].astype(np.int64), np.where(od == INT_MAX, np.iinfo(vdt).max, od)), \
                        f"{kind} row {k} against the oracle, depth_limit={limit}"


def check_schedules(monkeypatch, capfd, kind, size, n=65, seed=1):
    """never bottom-up, bottom-up from the first level and the default schedule: identical distances, valid predecessors,
    and the trace shows the directions each schedule asks for"""
    s, d, V, sym = edges(kind, size, seed)
    srcs = _pick_sources(s, V, n, seed)
    base = None
    for name, knobs in [("default", {})] + list(BFS_SCHEDULES.items()):
        h, g = _graph(monkeypatch, dict(knobs, BFS_TRACE="1"), s, d, symmetric=sym, vertices=np.arange(V, dtype=np.int32))
        capfd.readouterr()
        dist, pred, verts = ms_bfs(h, g, srcs)
        # the first batch starts at the hub; a batch whose sources have no out-edges (m_f = 0) stays top-down
        err = "\n".join(x for x in capfd.readouterr().err.splitlines() if x.startswith("ms-bfs batch 0 "))
        if name == "never-bottom-up":
            assert "ms-bfs batch 0 level 0 top-down" in err and "bottom-up" not in err, err
        if name == "bottom-up-from-the-first-level":
            assert "ms-bfs batch 0 level 0 bottom-up" in err and "top-down" not in err, err
        dist_id, pred_id = _by_id(verts, dist), _by_id(verts, pred)
        _assert_pred_rows(s, d, V, srcs, dist_id, pred_id)
        if base is None:
            base = dist_id
        assert np.array_equal(dist_id, base), name


def check_inputs(monkeypatch, size=400, seed=2):
    """isolated vertices from a vertices array, self-loops, multi-edges, an edgeless graph; duplicate sources, no
    sources, no predecessors"""
    rng = np.random.default_rng(seed)
    V = size
    s = rng.integers(0, V // 2, 3 * V).astype(np.int32)  # vertices V/2 .. V-1 only appear in the vertices array
    d = rng.integers(0, V // 2, 3 * V).astype(np.int32)
    s = np.concatenate([s, s[:50], np.arange(20, dtype=np.int32)])  # multi-edges and self-loops
    d = np.concatenate([d, d[:50], np.arange(20, dtype=np.int32)])
    for sym in (False, True):
        ss, dd = (np.concatenate([s, d]), np.concatenate([d, s])) if sym else (s, d)
        h, g = _graph(monkeypatch, {}, ss, dd, symmetric=sym, vertices=np.arange(V, dtype=np.int32))
        srcs = np.array([3, V - 1, 3, 7, V - 1], np.int64)
        dist, pred, verts = ms_bfs(h, g, srcs)
        assert np.array_equal(dist[0], dist[2]) and np.array_equal(dist[1], dist[4]), "duplicate sources"
        for k, src in enumerate(srcs.tolist()):
            rd, _, _ = single_bfs(h, g, src)
            assert np.array_equal(dist[k], rd), (sym, k)
        _assert_pred_rows(ss, dd, V, srcs, _by_id(verts, dist), _by_id(verts, pred))
        iso = _by_id(verts, dist)[1]
        assert iso[V - 1] == 0 and (np.delete(iso, V - 1) == INT_MAX).all(), "an isolated source reaches nothing"
        d0, p0, v0 = ms_bfs(h, g, np.zeros(0, np.int64))
        assert d0.shape == (0, V) and p0.shape == (0, V) and np.array_equal(v0, verts)
        d1, p1, _ = ms_bfs(h, g, srcs, compute_predecessors=False)
        assert p1 is None and np.array_equal(d1, dist)
        from cugraph_b200 import _capi
        import torch
        from cugraph_b200.pylibcugraph.algorithms import _paths_result
        from cugraph_b200.pylibcugraph.utils import View
        sv, res, err = View(torch.as_tensor(srcs.astype(np.int32)).cuda()), C.c_void_p(), C.c_void_p()
        code = _capi.lib().cugraph_b200_multi_source_bfs(h.ptr, g.ptr, sv.ptr, INT_MAX - 1, 0, C.byref(res), C.byref(err))
        _capi.check(code, err, "cugraph_b200_multi_source_bfs")
        sv.free()
        _, _, p_raw = _paths_result(h, res)
        assert p_raw.numel() == 0, "compute_predecessors=FALSE: predecessors of size 0"
    # no edges at all: every source reaches itself alone
    h, g = _graph(monkeypatch, {}, np.zeros(0, np.int32), np.zeros(0, np.int32), vertices=np.arange(50, dtype=np.int32))
    dist, pred, verts = ms_bfs(h, g, [4, 9])
    dist_id = _by_id(verts, dist)
    assert (dist_id[0, 4], dist_id[1, 9]) == (0, 0) and (dist_id == INT_MAX).sum() == 2 * 49 and (pred == -1).all()


def _call(h, g, sources_view, result=True):
    from cugraph_b200 import _capi
    res, err = C.c_void_p(), C.c_void_p()
    code = _capi.lib().cugraph_b200_multi_source_bfs(h.ptr, g.ptr, sources_view, INT_MAX - 1, 1,
                                                     C.byref(res) if result else None, C.byref(err))
    msg = ""
    if code != _capi.SUCCESS and err.value:
        msg = _capi.lib().cugraph_error_message(err).decode()
        _capi.lib().cugraph_error_free(err)
    return code, msg, res


def _extract_paths(h, g, res, source, dests):
    """(code, max path length, paths) of cugraph_extract_paths over a paths result"""
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View, copy_to_torch
    L = _capi.lib()
    sv = View(torch.tensor([source], dtype=torch.int32).cuda())
    dv = View(torch.as_tensor(np.asarray(dests, np.int32)).cuda())
    out, err = C.c_void_p(), C.c_void_p()
    code = L.cugraph_extract_paths(h.ptr, g.ptr, sv.ptr, res, dv.ptr, C.byref(out), C.byref(err))
    sv.free()
    dv.free()
    if code != _capi.SUCCESS:
        if err.value:
            L.cugraph_error_free(err)
        return code, 0, None
    n = int(L.cugraph_extract_paths_result_get_max_path_length(out))
    paths = copy_to_torch(h, L.cugraph_extract_paths_result_get_paths(out)).cpu().numpy().reshape(len(dests), n)
    L.cugraph_extract_paths_result_free(out)
    return code, n, paths


def check_errors(monkeypatch, size=300, seed=3):
    """an invalid source, the wrong source dtype, NULL arguments; cugraph_extract_paths on a one-row result (the paths of
    cugraph_bfs) and on a 64-row one (rejected)"""
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View
    s, d, V, sym = edges("random_sym", size, seed)
    h, g = _graph(monkeypatch, {}, s, d, symmetric=sym, vertices=np.arange(V, dtype=np.int32))
    L = _capi.lib()
    for bad, dtype, text in ((V + 5, torch.int32, "Found invalid vertex in the input sources"),
                             (-1, torch.int32, "Found invalid vertex in the input sources"),
                             (3, torch.int64, "vertex type of graph and sources must match")):
        sv = View(torch.tensor([1, bad], dtype=dtype).cuda())
        code, msg, _ = _call(h, g, sv.ptr)
        sv.free()
        assert code == _capi.INVALID_INPUT and text in msg, (bad, code, msg)
    code, msg, _ = _call(h, g, None)
    assert code == _capi.INVALID_INPUT, code
    sv = View(torch.tensor([1], dtype=torch.int32).cuda())
    code, msg, _ = _call(h, g, sv.ptr, result=False)
    assert code == _capi.INVALID_INPUT, code
    sv.free()
    dests = np.arange(0, V, 7)
    for source in (0, 11):
        sv = View(torch.tensor([source], dtype=torch.int32).cuda())
        code, _, res = _call(h, g, sv.ptr)
        sv.free()
        assert code == _capi.SUCCESS
        got = _extract_paths(h, g, res, source, dests)
        L.cugraph_paths_result_free(res)
        sv = View(torch.tensor([source], dtype=torch.int32).cuda())
        res, err = C.c_void_p(), C.c_void_p()
        _capi.check(L.cugraph_bfs(h.ptr, g.ptr, sv.ptr, 0, INT_MAX - 1, 1, 0, C.byref(res), C.byref(err)), err, "cugraph_bfs")
        sv.free()
        want = _extract_paths(h, g, res, source, dests)
        L.cugraph_paths_result_free(res)
        assert got[0] == want[0] == _capi.SUCCESS and got[1] == want[1]
        dist, _, verts = single_bfs(h, g, source)
        dist_id = _by_id(verts, dist[None])[0]
        for i, v in enumerate(dests.tolist()):  # the same endpoints and lengths; interior vertices may differ (any BFS tree)
            row = got[2][i]
            if dist_id[v] == INT_MAX:
                assert (row == -1).all()
            else:
                assert row[0] == source and row[dist_id[v]] == v and (row[dist_id[v] + 1:] == -1).all()
    sv = View(torch.as_tensor(_pick_sources(s, V, 64, seed).astype(np.int32)).cuda())
    code, _, res = _call(h, g, sv.ptr)
    sv.free()
    assert code == _capi.SUCCESS
    assert _extract_paths(h, g, res, 0, dests)[0] == _capi.INVALID_INPUT
    L.cugraph_paths_result_free(res)


def check_api(size=300, seed=4):
    """api.multi_source_bfs: the reference's frame against per-source api.bfs; the forms that are not built and the
    sources it rejects"""
    import pandas as pd
    from cugraph_b200 import api
    s, d, V, _ = edges("random", size, seed)
    for directed in (False, True):
        G = api.Graph(directed=directed).from_pandas_edgelist(pd.DataFrame({"source": s, "destination": d}))
        srcs = [5, 17, 0, 123]
        df = api.multi_source_bfs(G, srcs)
        assert list(df.columns) == ["vertex"] + [c for x in srcs for c in (f"distance_{x}", f"predecessor_{x}")]
        for x in srcs:
            one = api.bfs(G, x)
            m = pd.merge(df[["vertex", f"distance_{x}", f"predecessor_{x}"]], one, on="vertex")
            assert len(m) == len(df) == len(one)
            assert np.array_equal(m[f"distance_{x}"].to_numpy(), m["distance"].to_numpy())
            reached = m["distance"].to_numpy() != INT_MAX
            assert ((m[f"predecessor_{x}"].to_numpy() == -1) == (~reached | (m["vertex"].to_numpy() == x))).all()
        lim = api.multi_source_bfs(G, srcs[:2], depth_limit=1)
        assert (lim["distance_5"].to_numpy()[lim["distance_5"].to_numpy() != INT_MAX] <= 1).all()
    with pytest.raises(NotImplementedError):
        api.multi_source_bfs(G, [1], components=pd.DataFrame({"vertex": [1], "color": [0]}))
    with pytest.raises(NotImplementedError):
        api.multi_source_bfs(G, [1], offload=True)
    for bad in ([], [3, 4, 3], list(range(G.number_of_vertices() + 1))):
        with pytest.raises(ValueError):
            api.multi_source_bfs(G, bad)


# --------------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("kind,size", [("random", 3000), ("random_sym", 3000), ("rmat", 12), ("rmat_sym", 12),
                                       ("rmat", 16), ("rmat_sym", 16)])
def test_row_parity_gpu(monkeypatch, kind, size):
    check_rows(monkeypatch, kind, size, limits=LIMITS if size < 16 else (0,))


@pytest.mark.parametrize("kind", ["random", "random_sym"])
def test_rows_against_oracle_gpu(monkeypatch, kind):
    check_rows(monkeypatch, kind, 1000, n_sources=(70,), with_oracle=True)


@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_schedules_gpu(monkeypatch, capfd, kind):
    check_schedules(monkeypatch, capfd, kind, 14)


@pytest.mark.parametrize("store_transposed", [False, True])
@pytest.mark.parametrize("renumber", [True, False])
@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_layouts_gpu(monkeypatch, store_transposed, renumber, kind):
    check_rows(monkeypatch, kind, 12, n_sources=(65,), limits=(0, 2), store_transposed=store_transposed, renumber=renumber)


@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_int64_ids_and_offs64_gpu(monkeypatch, kind):
    check_rows(monkeypatch, kind, 12, n_sources=(65,), limits=(0, 2), vertex_dtype=np.int64)
    check_rows(monkeypatch, kind, 12, n_sources=(65,), limits=(0, 2), knobs=OFFS64)
    check_rows(monkeypatch, kind, 12, n_sources=(65,), limits=(0,), knobs=OFFS64, vertex_dtype=np.int64, store_transposed=True)


def test_inputs_gpu(monkeypatch):
    check_inputs(monkeypatch)


def test_errors_and_extract_paths_gpu(monkeypatch):
    check_errors(monkeypatch)


def test_api_gpu():
    check_api()


def test_rmat20_symmetric_64_sources_gpu(monkeypatch, capfd):
    """at this size Beamer's rule takes both directions and the in-edge view has hub rows (the warp-per-row path)"""
    s, d, V, _ = edges("rmat_sym", 20, 5)
    h, g = _graph(monkeypatch, {"BFS_TRACE": "1"}, s, d, symmetric=True, vertices=np.arange(V, dtype=np.int32))
    srcs = _pick_sources(s, V, 64, 5)
    capfd.readouterr()
    dist, pred, verts = ms_bfs(h, g, srcs)
    err = capfd.readouterr().err
    assert " top-down " in err and " bottom-up " in err, err
    for k, src in enumerate(srcs.tolist()):
        rd, _, _ = single_bfs(h, g, src)
        assert np.array_equal(dist[k], rd), k
    _assert_pred_rows(s, d, V, srcs, _by_id(verts, dist), _by_id(verts, pred))


def test_more_than_2_31_entries_gpu(monkeypatch):
    """65 sources x 2^25 vertices = 2.18e9 entries: the last rows (the second batch) against cugraph_bfs"""
    V = 1 << 25
    rng = np.random.default_rng(6)
    s = rng.integers(0, V, 1 << 21).astype(np.int32)
    d = rng.integers(0, V, 1 << 21).astype(np.int32)
    h, g = _graph(monkeypatch, {}, s, d, vertices=np.arange(V, dtype=np.int32))
    srcs = np.concatenate([s[:64], [V - 1]]).astype(np.int64)  # V - 1: most likely isolated
    import torch
    from cugraph_b200.traversal import multi_source_bfs
    dist, pred, verts = multi_source_bfs(h, g, torch.as_tensor(srcs.astype(np.int32)).cuda(), compute_predecessors=False)
    assert pred is None and tuple(dist.shape) == (65, V)
    for k in (63, 64):
        rd, _, _ = single_bfs(h, g, int(srcs[k]))
        assert np.array_equal(dist[k].cpu().numpy(), rd), k
    del dist
    torch.cuda.empty_cache()
