"""Vertex and edge betweenness centrality (cugraph_betweenness_centrality, cugraph_edge_betweenness_centrality through
cugraph_b200.pylibcugraph and cugraph_b200.api) on the GPU, against the CPU oracle of tests/betweenness_ref.py.

Batches hold up to 64 sources, so explicit lists of 1, 63, 64, 65 and 130 sources cover both sides of a batch boundary.
Values are compared with a relative tolerance of 1e-5 (FLOAT32 results) or 1e-10 (FLOAT64) and an absolute one scaled to
the largest value; the chain of diamonds, whose path counts pass 2^53, is compared with exact integer path counts.

The check_* functions are shared with tests/test_betweenness_cpu.py, which runs them on the CPU emulation of the library at
smaller sizes."""
import json
import os

import numpy as np
import pytest

from tests import betweenness_ref as ref
from tests.gpu_util import make_graph
from tests.test_multi_source_bfs_gpu import OFFS64, _graph, edges

pytestmark = pytest.mark.gpu

N_SOURCES = (1, 63, 64, 65, 130)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "edge_betweenness_golden.json")


def _dev(a, dtype):
    import torch
    return torch.as_tensor(np.asarray(a, dtype)).cuda()


def vertex_bc(h, g, V, sources, normalized, endpoints, vertex_dtype=np.int32):
    """library values by vertex id; sources None = every vertex"""
    from cugraph_b200 import pylibcugraph as plc
    k = None if sources is None else _dev(sources, vertex_dtype)
    verts, vals = plc.betweenness_centrality(h, g, k, None, normalized, endpoints, False)
    out = np.full(V, np.nan, vals.cpu().numpy().dtype)
    out[verts.cpu().numpy()] = vals.cpu().numpy()
    return out


def edge_bc(h, g, sources, normalized, vertex_dtype=np.int32):
    """(src, dst, values) sorted by (src, dst, value)"""
    from cugraph_b200 import pylibcugraph as plc
    k = None if sources is None else _dev(sources, vertex_dtype)
    s, d, v, ids = plc.edge_betweenness_centrality(h, g, k, None, normalized, False)
    assert ids is None
    s, d, v = s.cpu().numpy().astype(np.int64), d.cpu().numpy().astype(np.int64), v.cpu().numpy()
    o = np.lexsort((v, d, s))
    return s[o], d[o], v[o]


def _close(got, want, dtype):
    rtol = 1e-5 if dtype == np.float32 else 1e-10
    fin = np.isfinite(want)
    assert (np.isnan(got) == np.isnan(want)).all(), "NaN positions differ"
    scale = max(float(np.abs(want[fin]).max()) if fin.any() else 0.0, 1e-30)
    np.testing.assert_allclose(got[fin], want[fin], rtol=rtol, atol=rtol * scale)


def _pick(V, n, seed):
    rng = np.random.default_rng(seed)
    return rng.permutation(V)[:n].astype(np.int64)


def check_vertex(s, d, V, sym, h, g, n_sources=N_SOURCES, full=True, dtype=np.float32, vertex_dtype=np.int32, seed=0):
    """every normalized x endpoints combination, full sources and lists of n_sources"""
    lists = ([None] if full else []) + [_pick(V, n, seed + n) for n in n_sources if n <= V]
    for srcs in lists:
        for norm in (False, True):
            for ep in (False, True):
                got = vertex_bc(h, g, V, srcs, norm, ep, vertex_dtype)
                want = ref.betweenness(s, d, V, srcs, norm, ep, sym, dtype)
                _close(got, want, dtype)


def check_edges(s, d, V, sym, h, g, n_sources=N_SOURCES, full=True, dtype=np.float32, vertex_dtype=np.int32, seed=0):
    lists = ([None] if full else []) + [_pick(V, n, seed + n) for n in n_sources if n <= V]
    for srcs in lists:
        for norm in (False, True):
            gs, gd, gv = edge_bc(h, g, srcs, norm, vertex_dtype)
            want = ref.edge_betweenness(s, d, V, srcs, norm, sym, dtype)
            o = np.lexsort((want, np.asarray(d, np.int64), np.asarray(s, np.int64)))
            assert np.array_equal(gs, np.asarray(s, np.int64)[o]) and np.array_equal(gd, np.asarray(d, np.int64)[o])
            _close(gv, want[o], dtype)


def check_graph(monkeypatch, kind, size, n_sources=N_SOURCES, full=True, knobs=None, seed=0, **kw):
    s, d, V, sym = edges(kind, size, seed)
    vdt = kw.get("vertex_dtype", np.int32)
    h, g = _graph(monkeypatch, knobs or {}, s, d, symmetric=sym, vertices=np.arange(V, dtype=vdt), **kw)
    check_vertex(s, d, V, sym, h, g, n_sources, full, vertex_dtype=vdt, seed=seed)
    check_edges(s, d, V, sym, h, g, n_sources[:2], full, vertex_dtype=vdt, seed=seed)


def check_layouts(monkeypatch, kind, size, n=65):
    """both storage orientations, renumbering on and off, INT64 ids, 64-bit offsets"""
    for st in (False, True):
        for rn in (True, False):
            check_graph(monkeypatch, kind, size, (n,), False, store_transposed=st, renumber=rn)
    check_graph(monkeypatch, kind, size, (n,), False, vertex_dtype=np.int64, renumber=False)
    check_graph(monkeypatch, kind, size, (n,), False, knobs=OFFS64, store_transposed=True)
    check_graph(monkeypatch, kind, size, (n,), False, knobs=OFFS64, vertex_dtype=np.int64)


def check_special(monkeypatch):
    """isolated and unreached vertices, self-loops, multi-edges, an edgeless graph"""
    s = np.array([0, 1, 1, 2, 2, 3, 3, 5, 5, 6, 7], np.int32)  # 4 and 9 isolated; 3 -> 3 self-loop; 2 -> 3 twice
    d = np.array([1, 2, 2, 3, 3, 3, 0, 6, 6, 7, 5], np.int32)
    V = 10
    for sym in (False, True):
        ss, dd = (np.concatenate([s, d]), np.concatenate([d, s])) if sym else (s, d)
        h, g = make_graph(ss, dd, symmetric=sym, vertices=np.arange(V, dtype=np.int32))
        check_vertex(ss, dd, V, sym, h, g, (1, 3, 10))
        check_edges(ss, dd, V, sym, h, g, (1, 3, 10))
    h, g = make_graph(np.zeros(0, np.int32), np.zeros(0, np.int32), vertices=np.arange(5, dtype=np.int32))
    for ep in (False, True):
        _close(vertex_bc(h, g, 5, None, False, ep), ref.betweenness([], [], 5, None, False, ep), np.float32)
    assert edge_bc(h, g, None, True)[0].size == 0


def check_path(n):
    """a directed path of n vertices: n - 1 levels from vertex 0"""
    s = np.arange(n - 1, dtype=np.int32)
    d = s + 1
    h, g = make_graph(s, d, vertices=np.arange(n, dtype=np.int32))
    srcs = np.array([0, 1, n // 2], np.int64)
    for ep in (False, True):
        _close(vertex_bc(h, g, n, srcs, False, ep), ref.betweenness(s, d, n, srcs, False, ep), np.float32)
    gs, gd, gv = edge_bc(h, g, srcs, False)
    _close(gv, ref.edge_betweenness(s, d, n, srcs, False), np.float32)


def check_diamonds(n_diamonds=62):
    """a chain of diamonds a -> {b, c} -> a': 2^k shortest paths reach the k-th joint, past 2^53 for k > 53.  FLOAT64, and
    the oracle's path counts are exact integers: the values agree to 1e-12 relative"""
    s, d = [], []
    for k in range(n_diamonds):
        a, b, c, z = 3 * k, 3 * k + 1, 3 * k + 2, 3 * k + 3
        s += [a, a, b, c]
        d += [b, c, z, z]
    V = 3 * n_diamonds + 1
    s, d = np.array(s, np.int32), np.array(d, np.int32)
    h, g = make_graph(s, d, weights=np.ones(s.size), weight_dtype=np.float64, vertices=np.arange(V, dtype=np.int32))
    srcs = np.array([0, 3], np.int64)
    bc, _, sig = ref.brandes(s, d, V, srcs, exact=True)
    assert max(sig[0]) == 2**n_diamonds
    got = vertex_bc(h, g, V, srcs, False, False)
    want = ref.betweenness(s, d, V, srcs, False, False, dtype=np.float64, exact=True)
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=0)
    gs, gd, gv = edge_bc(h, g, srcs, False)
    we = ref.edge_betweenness(s, d, V, srcs, False, dtype=np.float64)
    o = np.lexsort((we, d.astype(np.int64), s.astype(np.int64)))
    np.testing.assert_allclose(gv, we[o], rtol=1e-12, atol=0)


def check_float64(monkeypatch):
    s, d, V, sym = edges("random_sym", 200, 3)
    h, g = make_graph(s, d, weights=np.ones(s.size), weight_dtype=np.float64, symmetric=sym,
                      vertices=np.arange(V, dtype=np.int32))
    check_vertex(s, d, V, sym, h, g, (65,), dtype=np.float64)
    check_edges(s, d, V, sym, h, g, (65,), dtype=np.float64)
    assert vertex_bc(h, g, V, None, True, False).dtype == np.float64


def check_deterministic(kind, size):
    """two identical calls give bit-identical values"""
    s, d, V, sym = edges(kind, size, 1)
    h, g = make_graph(s, d, symmetric=sym, vertices=np.arange(V, dtype=np.int32))
    srcs = _pick(V, min(V, 130), 5)
    a, b = vertex_bc(h, g, V, srcs, True, False), vertex_bc(h, g, V, srcs, True, False)
    assert a.tobytes() == b.tobytes()
    ea, eb = edge_bc(h, g, srcs, True), edge_bc(h, g, srcs, True)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(ea, eb))


def check_errors():
    import ctypes as C
    from cugraph_b200 import _capi
    from cugraph_b200 import pylibcugraph as plc
    s = np.array([0, 1, 2], np.int32)
    h, g = make_graph(s, s + 1, vertices=np.arange(4, dtype=np.int32))
    for fn in (lambda k: plc.betweenness_centrality(h, g, k, None, True, False, False),
               lambda k: plc.edge_betweenness_centrality(h, g, k, None, True, False)):
        with pytest.raises(Exception, match="sources have invalid vertex IDs"):
            fn(_dev([0, 7], np.int32))
        with pytest.raises(Exception, match="vertex type of graph and vertex_list must match"):
            fn(_dev([0], np.int64))
        with pytest.raises(Exception, match="should not exceed the number of vertices"):
            fn(5)
    L = _capi.lib()
    err, res = C.c_void_p(), C.c_void_p()
    bad = _dev([9], np.int32)
    sv = L.cugraph_type_erased_device_array_view_create(C.c_void_p(bad.data_ptr()), 1, 4)  # 4: INT32
    code = L.cugraph_betweenness_centrality(h.ptr, g.ptr, sv, 1, 0, 0, C.byref(res), C.byref(err))
    assert code == _capi.INVALID_INPUT
    L.cugraph_error_free(err)
    L.cugraph_type_erased_device_array_view_free(sv)


def check_select_random_vertices():
    """distinct vertices, the same for the same seed, every vertex when asked for all"""
    from cugraph_b200 import pylibcugraph as plc
    s, d, V, sym = edges("random", 300, 0)
    h, g = make_graph(s, d, vertices=np.arange(V, dtype=np.int32))
    a = plc.select_random_vertices(h, g, 7, 50).cpu().numpy()
    b = plc.select_random_vertices(h, g, 7, 50).cpu().numpy()
    c = plc.select_random_vertices(h, g, 8, 50).cpu().numpy()
    assert np.unique(a).size == 50 and a.min() >= 0 and a.max() < V
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    assert np.array_equal(np.sort(plc.select_random_vertices(h, g, 1, V).cpu().numpy()), np.arange(V))


def check_api():
    """pylibcugraph k as an int and as an array; api frames; weight raises"""
    import pandas as pd
    from cugraph_b200 import api
    from cugraph_b200 import pylibcugraph as plc
    s, d, V, _ = edges("random", 120, 2)
    s, d = np.concatenate([s, np.arange(V, dtype=np.int32)]), np.concatenate([d, (np.arange(V, dtype=np.int32) + 1) % V])
    h, g = make_graph(s, d, vertices=np.arange(V, dtype=np.int32))
    picked = plc.select_random_vertices(h, g, 3, 20).cpu().numpy()
    verts, vals = plc.betweenness_centrality(h, g, 20, 3, True, False, False)
    by_int = np.zeros(V, np.float32)
    by_int[verts.cpu().numpy()] = vals.cpu().numpy()
    _close(by_int, ref.betweenness(s, d, V, picked, True, False), np.float32)
    s2, d2, v2, ids = plc.edge_betweenness_centrality(h, g, 20, 3, True, False)
    assert ids is None and s2.shape[0] == s.size
    G = api.Graph(directed=True).from_pandas_edgelist(pd.DataFrame({"source": s, "destination": d}))
    df = api.betweenness_centrality(G)
    assert list(df.columns) == ["vertex", "betweenness_centrality"] and df["betweenness_centrality"].dtype == np.float64
    got = np.zeros(V)
    got[df["vertex"].to_numpy()] = df["betweenness_centrality"].to_numpy()
    _close(got.astype(np.float32), ref.betweenness(s, d, V, None, True, False), np.float32)
    lst = [3, 17, 40]
    df2 = api.betweenness_centrality(G, k=lst, normalized=False, endpoints=True, result_dtype=np.float32)
    assert df2["betweenness_centrality"].dtype == np.float32
    got = np.zeros(V, np.float32)
    got[df2["vertex"].to_numpy()] = df2["betweenness_centrality"].to_numpy()
    _close(got, ref.betweenness(s, d, V, lst, False, True), np.float32)
    with pytest.raises(NotImplementedError):
        api.betweenness_centrality(G, weight="w")
    with pytest.raises(NotImplementedError):
        api.edge_betweenness_centrality(G, weight="w")
    de = api.edge_betweenness_centrality(G, k=lst)
    assert list(de.columns) == ["src", "dst", "betweenness_centrality"] and len(de) == s.size
    U = api.Graph(directed=False).from_pandas_edgelist(pd.DataFrame({"source": s, "destination": d}))
    du = api.edge_betweenness_centrality(U)
    assert (du["src"] <= du["dst"]).all() and len(du) < s.size


def check_golden():
    """the expected scores of the reference's pylibcugraph edge betweenness test (toy graph, every source, normalized)"""
    gd = json.load(open(GOLDEN))
    s, d = np.array(gd["src"], np.int32), np.array(gd["dst"], np.int32)
    h, g = make_graph(s, d, store_transposed=gd["store_transposed"], renumber=False)
    want = np.zeros(len(s), np.float32)
    want[np.array(gd["result_edge_ids"])] = gd["result_scores"]
    gs, gdd, gv = edge_bc(h, g, None, gd["normalized"])
    o = np.lexsort((want, d.astype(np.int64), s.astype(np.int64)))
    assert np.array_equal(gs, s[o]) and np.array_equal(gdd, d[o])
    np.testing.assert_allclose(gv, want[o], rtol=gd["rel_tol"])


# ---- the GPU tests
@pytest.mark.parametrize("kind", ["random", "random_sym"])
def test_random_graphs(monkeypatch, kind):
    check_graph(monkeypatch, kind, 400)


@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_rmat_graphs(monkeypatch, kind):
    check_graph(monkeypatch, kind, 10, full=False)


def test_layouts(monkeypatch):
    check_layouts(monkeypatch, "rmat", 9)
    check_layouts(monkeypatch, "rmat_sym", 9)


def test_special_graphs(monkeypatch):
    check_special(monkeypatch)


def test_long_path():
    check_path(10_000)


def test_diamond_chain_beyond_2_53():
    check_diamonds()


def test_float64(monkeypatch):
    check_float64(monkeypatch)


def test_bit_identical_repeats():
    check_deterministic("rmat_sym", 12)


def test_errors():
    check_errors()


def test_select_random_vertices():
    check_select_random_vertices()


def test_api():
    check_api()


def test_pylibcugraph_golden():
    check_golden()


def test_rmat20_130_sources(monkeypatch):
    """symmetrised RMAT-20 (about 33.5 M directed edges) from 130 sources, vertex and edge values against the oracle"""
    s, d, V, sym = edges("rmat_sym", 20, 0)
    h, g = make_graph(s, d, symmetric=sym, vertices=np.arange(V, dtype=np.int32))
    srcs = _pick(V, 130, 11)
    _close(vertex_bc(h, g, V, srcs, True, False), ref.betweenness(s, d, V, srcs, True, False, sym), np.float32)
