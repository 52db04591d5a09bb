"""The paths the library only picks by graph size or orientation, forced with the schedule knobs on small RMAT graphs and
checked against the CPU oracle and against the default run of the same graph.

- offs64: CUGRAPH_B200_OFFS64_MIN_EDGES=0 gives every graph 64-bit row offsets, which by default only graphs of 2^31 or
  more edges get (the int64_t instantiations of BFS, SSSP with its own schedule, the plain sweep of PageRank / Katz / HITS /
  eigenvector, WCC, degrees, the expensive input check).  Together with CUGRAPH_B200_ADVANCE_SPLIT_EDGES it also takes
  the advance in halves that such graphs need.
- The piece-stream sweep on Katz, HITS, eigenvector and on CSR graphs, where it runs over a re-sorted view (row_vertex).
- SSSP and BFS under forced schedules.

Distances are bit-exact (the min/add fixpoint does not depend on the order of the relaxations), predecessors are checked
with the oracle's validity predicates and, for SSSP, by walking every predecessor chain back to the source.

The check_* functions are shared with tests/test_offsets64_cpu.py, which runs them on the CPU emulation of the library.
There they run at a smaller scale: the emulation executes the threads of a launch one after the other."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle.rmat import rmat_edgelist
from tests.gpu_util import by_vertex, make_graph
from tests.test_pagerank_gpu import REL, _run as _pagerank

pytestmark = pytest.mark.gpu

INT_MAX = 2**31 - 1
OFFS64 = {"OFFS64_MIN_EDGES": "0"}
PLAIN_SWEEP = {"SWEEP_MIN_EDGES": str(1 << 40)}
EMULATED_MAX_SCALE = 10
# PageRank on 64-bit offsets against the 32-bit plain sweep of the same graph: the same kernels but for the offset type.
# Measured on an H100 80GB HBM3 (400 W power limit), RMAT-16, 30 iterations, CSC unweighted and weighted and CSR: the scores
# were identical (0 ulp).  The bound leaves one ulp because rows split over several CTAs add their fp64 partial sums with
# atomics, in no fixed order, and such a sum can round to the neighbouring fp32 value.
PAGERANK_OFFS64_MAX_ULPS = 1


def _scale(scale):
    from cugraph_b200 import _capi
    return min(scale, EMULATED_MAX_SCALE) if _capi.emulated() else scale


def _graph(monkeypatch, knobs, *args, **kw):
    """make_graph with CUGRAPH_B200_<knob> set while its handle is created (the handle reads the knobs once; lazily built
    views of the graph follow the handle that the algorithm is called with, which is this one)"""
    for k, v in knobs.items():
        monkeypatch.setenv("CUGRAPH_B200_" + k, v)
    try:
        return make_graph(*args, **kw)
    finally:
        for k in knobs:
            monkeypatch.delenv("CUGRAPH_B200_" + k)


def _rmat(scale, seed, symmetric=False):
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed)
    s, d = np.asarray(s, np.int32), np.asarray(d, np.int32)
    if symmetric:
        s, d = np.concatenate([s, d]), np.concatenate([d, s])
    return s, d, 1 << scale


def _sym_weights(n_half, seed, wdtype):
    w = np.random.default_rng(seed).random(n_half).astype(wdtype)
    return np.concatenate([w, w])


def _compare_sweeps(h, g):
    from cugraph_b200 import _capi
    out = (C.c_double * 8)()
    err = C.c_void_p()
    f = _capi.lib().cugraph_b200_debug_compare_sweeps
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    _capi.check(f(h.ptr, g.ptr, C.cast(out, C.c_void_p), C.byref(err)), err, "cugraph_b200_debug_compare_sweeps")
    return list(out)


def _assert_predecessor_tree(dist, pred, source, unreached):
    """every reached vertex's predecessor chain ends at the source (no cycle), distances never increase along it"""
    V = dist.size
    reached = dist != unreached
    assert (pred[~reached] == -1).all()
    inner = reached.copy()
    inner[source] = False
    assert pred[source] == -1 and (pred[inner] >= 0).all()
    assert (dist[pred[inner]] <= dist[inner]).all()
    jump = np.where(inner, pred, np.arange(V))        # the source and the unreached vertices point at themselves
    for _ in range(int(np.ceil(np.log2(max(V, 2)))) + 1):
        jump = jump[jump]
    bad = np.flatnonzero(reached & (jump != source))
    assert bad.size == 0, f"predecessor cycle reached from vertex {bad[:5].tolist()}"


# ------------------------------------------------------------------------------------------------------------ BFS
def _bfs(h, g, sources, do, depth_limit=0, vertex_dtype=np.int32):
    import torch
    from cugraph_b200 import pylibcugraph as plc
    dist, pred, verts = plc.bfs(h, g, torch.as_tensor(np.asarray(sources, vertex_dtype)).cuda(), do, depth_limit, True, False)
    return verts, dist, pred


def check_bfs(monkeypatch, knobs, scale, directions=(False, True), depth_limit=True):
    """top-down and / or direction-optimising BFS from a hub, two other vertices, three at once and an isolated vertex,
    with and without a depth limit"""
    s, d, V = _rmat(_scale(scale), seed=400 + scale, symmetric=True)
    deg = np.bincount(s, minlength=V)
    iso = int(np.flatnonzero(deg == 0)[0])
    others = np.random.default_rng(scale).choice(np.flatnonzero(deg > 0), 3, replace=False).tolist()
    source_sets = [[int(deg.argmax())], others[:1], others, [iso]]
    hk, gk = _graph(monkeypatch, knobs, s, d, symmetric=True, vertices=np.arange(V, dtype=np.int32))
    h0, g0 = _graph(monkeypatch, {}, s, d, symmetric=True, vertices=np.arange(V, dtype=np.int32))
    csr = oracle.coo_to_csx(s, d, V)
    for do in directions:
        for srcs in source_sets:
            for limit in ((0, 2) if depth_limit else (0,)):
                ref_d, _ = oracle.bfs(s, d, V, srcs, depth_limit=limit or None, csr=csr)
                verts, dist, pred = _bfs(hk, gk, srcs, do, limit)
                got_d, got_p = by_vertex(verts, dist, V), by_vertex(verts, pred, V)
                case = f"direction_optimizing={do} sources={srcs} depth_limit={limit}"
                assert np.array_equal(got_d, ref_d), case
                assert oracle.check_bfs_predecessors(s, d, V, got_d, got_p, srcs), case
                verts, dist, _ = _bfs(h0, g0, srcs, do, limit)
                assert np.array_equal(got_d, by_vertex(verts, dist, V)), case


# ----------------------------------------------------------------------------------------------------------- SSSP
def _sssp(h, g, source, cutoff=float("inf"), pred=True):
    from cugraph_b200 import pylibcugraph as plc
    return plc.sssp(h, g, source, cutoff, pred, False)


def _check_sssp_graph(monkeypatch, knobs, s, d, w, V, sources, cutoff=True, no_pred=True):
    wd = w.dtype.type
    use_float = wd == np.float32
    unreached = np.finfo(wd).max
    hk, gk = _graph(monkeypatch, knobs, s, d, w, symmetric=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=wd)
    h0, g0 = _graph(monkeypatch, {}, s, d, w, symmetric=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=wd)
    csr = oracle.coo_to_csx(s, d, V, w)
    for src in sources:
        case = f"{wd.__name__} source={src}"
        ref_d, _ = oracle.sssp(s, d, w, V, src, use_float=use_float, csr=csr)
        verts, dist, pred = _sssp(hk, gk, src)
        got_d, got_p = by_vertex(verts, dist, V), by_vertex(verts, pred, V)
        assert np.array_equal(got_d.astype(np.float64), ref_d), case
        assert oracle.check_sssp_predecessors(s, d, w, V, got_d.astype(np.float64), got_p, src), case
        _assert_predecessor_tree(got_d, got_p, src, unreached)
        verts, dist, _ = _sssp(h0, g0, src)
        assert np.array_equal(got_d, by_vertex(verts, dist, V)), case
        if no_pred:
            verts, dist, _ = _sssp(hk, gk, src, pred=False)
            assert np.array_equal(by_vertex(verts, dist, V).astype(np.float64), ref_d), case + " without predecessors"
        if cutoff:
            reach = ref_d[ref_d < unreached]
            co = float(np.quantile(reach, 0.3))
            ref_c, _ = oracle.sssp(s, d, w, V, src, cutoff=co, use_float=use_float, csr=csr)
            verts, dist, pred = _sssp(hk, gk, src, cutoff=co)
            got_c = by_vertex(verts, dist, V)
            assert np.array_equal(got_c.astype(np.float64), ref_c), case + f" cutoff={co}"
            assert oracle.check_sssp_predecessors(s, d, w, V, got_c.astype(np.float64), by_vertex(verts, pred, V), src)


def check_sssp(monkeypatch, knobs, scale, wdtypes=(np.float32, np.float64), cutoff=True, no_pred=True):
    """weighted symmetric RMAT from a hub and from another vertex: float32 with predecessors (the packed word), float32
    without, float64 (predecessors from the distance fixpoint), a cutoff"""
    s, d, V = _rmat(_scale(scale), seed=500 + scale, symmetric=True)
    deg = np.bincount(s, minlength=V)
    sources = [int(deg.argmax()), int(np.flatnonzero(deg > 0)[-1])]
    for wd in wdtypes:
        w = _sym_weights(s.size // 2, scale, wd)
        _check_sssp_graph(monkeypatch, knobs, s, d, w, V, sources,
                          cutoff=cutoff and wd == np.float32, no_pred=no_pred and wd == np.float32)


def check_sssp_zero_weights(monkeypatch, knobs, wdtype):
    """the graph of test_sssp_zero_weight_predecessors_form_a_tree: zero-weight edges both ways, a zero-weight cycle and a
    weight absorbed by rounding (1e8 + 1 == 1e8 in float, 1e16 + 1 == 1e16 in double)"""
    r = np.random.default_rng(3)
    V = 4000
    hs = r.integers(0, V, 16000).astype(np.int32)
    hd = r.integers(0, V, 16000).astype(np.int32)
    hw = np.where(r.random(16000) < 0.5, 0.0, r.random(16000))
    big = 1e8 if wdtype == np.float32 else 1e16
    extra = [(6, 7, 0.0), (7, 8, 0.0), (8, 9, 0.0), (9, 7, 0.0), (0, 3990, big), (3990, 3991, 1.0), (3991, 3992, 1.0)]
    hs = np.concatenate([hs, np.array([e[0] for e in extra], np.int32)])
    hd = np.concatenate([hd, np.array([e[1] for e in extra], np.int32)])
    hw = np.concatenate([hw, [e[2] for e in extra]]).astype(wdtype)
    s, d, w = np.concatenate([hs, hd]), np.concatenate([hd, hs]), np.concatenate([hw, hw])
    _check_sssp_graph(monkeypatch, knobs, s, d, w, V, [0, 7], cutoff=False, no_pred=False)


# ------------------------------------------------------------------------------------------------------- PageRank
def check_pagerank_offs64(monkeypatch, scale, store_transposed, weighted):
    """PageRank on 64-bit offsets with the piece stream allowed at any size: the stream refuses such graphs, PageRank takes
    the plain sweep.  Against the fp64 oracle and the 32-bit plain sweep of the same graph; returns the largest difference
    between the two in fp32 ulps"""
    from cugraph_b200 import _capi
    s, d, V = _rmat(_scale(scale), seed=600 + scale)
    w = np.random.default_rng(7).random(s.size).astype(np.float32) + 0.25 if weighted else None
    kw = dict(store_transposed=store_transposed, vertices=np.arange(V, dtype=np.int32))
    hk, gk = _graph(monkeypatch, {**OFFS64, "SWEEP_MIN_EDGES": "0"}, s, d, w, **kw)
    h0, g0 = _graph(monkeypatch, PLAIN_SWEEP, s, d, w, **kw)
    verts, vals, _ = _pagerank(hk, gk, 0.85, 0.0, 30)
    got = by_vertex(verts, vals, V)
    ref, _, _ = oracle.pagerank(s, d, V, None if w is None else w.astype(np.float64), alpha=0.85, epsilon=0.0, max_iterations=30)
    np.testing.assert_allclose(got, ref, rtol=REL, atol=1e-12)
    verts, vals, _ = _pagerank(h0, g0, 0.85, 0.0, 30)
    base = by_vertex(verts, vals, V)
    ulps = float((np.abs(got - base) / np.spacing(np.maximum(np.abs(got), np.abs(base)))).max())
    print(f"PageRank RMAT-{_scale(scale)} store_transposed={store_transposed} weighted={weighted}: 64-bit against 32-bit "
          f"offsets, largest difference {ulps:.0f} fp32 ulp")
    assert ulps <= PAGERANK_OFFS64_MAX_ULPS, ulps
    with pytest.raises(_capi.CugraphError) as e:   # the row-by-row sweep comparison is 32-bit only
        _compare_sweeps(hk, gk)
    assert e.value.code == _capi.NOT_IMPLEMENTED
    return ulps


def check_pagerank_stream(monkeypatch, knobs, scale, weighted):
    """PageRank on a CSR graph: the piece stream runs over the re-sorted transpose (pull_alt, rows through row_vertex);
    against the fp64 oracle and, row by row, against the plain sweep"""
    s, d, V = _rmat(_scale(scale), seed=700 + scale)
    w = np.random.default_rng(8).random(s.size).astype(np.float32) + 0.25 if weighted else None
    h, g = _graph(monkeypatch, knobs, s, d, w, store_transposed=False, vertices=np.arange(V, dtype=np.int32))
    verts, vals, _ = _pagerank(h, g, 0.85, 0.0, 30)
    ref, _, _ = oracle.pagerank(s, d, V, None if w is None else w.astype(np.float64), alpha=0.85, epsilon=0.0, max_iterations=30)
    np.testing.assert_allclose(by_vertex(verts, vals, V), ref, rtol=REL, atol=1e-12)
    out = _compare_sweeps(h, g)
    assert out[0] < 2e-6 and out[4] < 2e-6 and out[3] == 0 and out[7] == 0, out


# ------------------------------------------------------------------------------------------ Katz, HITS, eigenvector
def check_siblings(monkeypatch, knobs, scale, weighted=True):
    """Katz (weighted), eigenvector (weighted), HITS (ignores the weights) with store_transposed True and False, at the
    tolerances of test_siblings_gpu.py"""
    from cugraph_b200 import pylibcugraph as plc
    s, d, V = _rmat(_scale(scale), seed=800 + scale)
    w = np.random.default_rng(1).random(s.size).astype(np.float32) + 0.5 if weighted else None
    for st in (True, False):
        h, g = _graph(monkeypatch, knobs, s, d, w, store_transposed=st, vertices=np.arange(V, dtype=np.int32))
        verts, hubs, auth = plc.hits(h, g, 1e-7, 500, None, None, True, False)
        rh, ra, _, _ = oracle.hits(s, d, V, epsilon=1e-7)
        np.testing.assert_allclose(by_vertex(verts, hubs, V), rh, rtol=2e-3, atol=1e-9)
        np.testing.assert_allclose(by_vertex(verts, auth, V), ra, rtol=2e-3, atol=1e-9)
        if not st:
            continue
        alpha = 0.5 / (np.bincount(d).max() * (float(w.max()) if weighted else 1.0))
        verts, vals = plc.katz_centrality(h, g, None, alpha, 1.0, 1e-5, 500, False)
        ref, _ = oracle.katz(s, d, V, w, alpha=alpha, beta=1.0, epsilon=1e-5, dtype=np.float32)
        np.testing.assert_allclose(by_vertex(verts, vals, V), ref, rtol=2e-5)
        verts, vals = plc.eigenvector_centrality(h, g, 1e-7, 1000, False)
        ref, _ = oracle.eigenvector(s, d, V, w, epsilon=1e-7, max_iterations=1000)
        np.testing.assert_allclose(by_vertex(verts, vals, V), ref, rtol=2e-3, atol=1e-8)


# -------------------------------------------------------------------------- WCC, degrees, extract_paths, CSR, int64
def _bfs_extract_paths(h, g, source, dests):
    """cugraph_extract_paths on the BFS result from `source`: (vertices, distances, paths[len(dests), max length])"""
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View, copy_to_torch
    L = _capi.lib()
    sv = View(torch.tensor([source], dtype=torch.int32).cuda())
    dv = View(torch.as_tensor(np.asarray(dests, np.int32)).cuda())
    res, out, err = C.c_void_p(), C.c_void_p(), C.c_void_p()
    h.order_after_caller()
    _capi.check(L.cugraph_bfs(h.ptr, g.ptr, sv.ptr, 0, INT_MAX - 1, 1, 0, C.byref(res), C.byref(err)), err, "cugraph_bfs")
    verts = copy_to_torch(h, L.cugraph_paths_result_get_vertices(res))
    dist = copy_to_torch(h, L.cugraph_paths_result_get_distances(res))
    code = L.cugraph_extract_paths(h.ptr, g.ptr, sv.ptr, res, dv.ptr, C.byref(out), C.byref(err))
    L.cugraph_paths_result_free(res)
    _capi.check(code, err, "cugraph_extract_paths")
    n = int(L.cugraph_extract_paths_result_get_max_path_length(out))
    paths = copy_to_torch(h, L.cugraph_extract_paths_result_get_paths(out)).cpu().numpy().reshape(len(dests), n)
    L.cugraph_extract_paths_result_free(out)
    sv.free()
    dv.free()
    return verts, dist, paths


def check_structure(monkeypatch, knobs, scale):
    """WCC (same partition as the oracle), in- and out-degrees (exact) and extract_paths (every row a path of graph edges
    from the source, as long as the BFS distance) on a symmetric graph with isolated vertices"""
    from cugraph_b200 import pylibcugraph as plc
    s, d, V = _rmat(_scale(scale), seed=900 + scale, symmetric=True)
    h, g = _graph(monkeypatch, knobs, s, d, symmetric=True, vertices=np.arange(V, dtype=np.int32), do_expensive_check=True)
    verts, labels = plc.weakly_connected_components(h, g, None, None, None, None, False)
    ref = oracle.wcc(s, d, V)
    got = by_vertex(verts, labels, V)
    assert len(set(zip(ref.tolist(), got.tolist()))) == len(set(ref.tolist())) == len(set(got.tolist()))
    v, din, dout = plc.degrees(h, g, None, False)
    v = v.cpu().numpy()
    assert np.array_equal(din.cpu().numpy(), np.bincount(d, minlength=V)[v])
    assert np.array_equal(dout.cpu().numpy(), np.bincount(s, minlength=V)[v])
    deg = np.bincount(s, minlength=V)
    source = int(deg.argmax())
    r = np.random.default_rng(2)
    dests = np.concatenate([r.choice(np.flatnonzero(deg > 0), 100), np.flatnonzero(deg == 0)[:3], [source]])
    verts, dist, paths = _bfs_extract_paths(h, g, source, dests)
    dist = by_vertex(verts, dist, V)
    ref_d, _ = oracle.bfs(s, d, V, [source])
    assert np.array_equal(dist, ref_d)
    _assert_bfs_paths(s, d, V, source, dests, dist, paths)


def _assert_bfs_paths(s, d, V, source, dests, dist, paths):
    """extract_paths rows against the BFS distances: the row length is 1 + the largest reached distance of a destination;
    a reached destination's row is a chain of graph edges from the source, one hop per BFS level, padded with -1; an
    unreached destination's row is all -1"""
    assert paths.shape[1] == 1 + int(dist[dests][dist[dests] < INT_MAX].max())
    keys = np.unique(s.astype(np.int64) * V + d)
    for row, t in zip(paths, np.asarray(dests).tolist()):
        if dist[t] == INT_MAX:
            assert (row == -1).all()
            continue
        n = int(dist[t]) + 1
        assert row[0] == source and row[n - 1] == t and (row[n:] == -1).all()
        hop = row[:n - 1].astype(np.int64) * V + row[1:n]
        pos = np.minimum(np.searchsorted(keys, hop), keys.size - 1)   # keys are sorted: a lookup, not np.isin's sort
        assert (keys[pos] == hop).all() and np.array_equal(dist[row[:n]], np.arange(n))


def check_csr_input(monkeypatch, knobs):
    """a graph given as CSR arrays (cugraph_graph_create_sg_from_csr, with the expensive input check): BFS and SSSP"""
    rng = np.random.default_rng(12)
    V, E = 3000, 30000
    s = rng.integers(0, V, E).astype(np.int32)
    d = rng.integers(0, V, E).astype(np.int32)
    w = rng.random(E).astype(np.float32)
    order = np.lexsort((d, s))
    s, d, w = s[order], d[order], w[order]
    offs = np.concatenate([[0], np.cumsum(np.bincount(s, minlength=V))]).astype(np.int32)
    h, g = _graph(monkeypatch, knobs, offs, d, w, input_array_format="CSR", renumber=False, do_expensive_check=True)
    verts, dist, pred = _sssp(h, g, 5)
    ref_d, _ = oracle.sssp(s, d, w, V, 5)
    got_d = by_vertex(verts, dist, V).astype(np.float64)
    assert np.array_equal(got_d, ref_d)
    assert oracle.check_sssp_predecessors(s, d, w, V, got_d, by_vertex(verts, pred, V), 5)
    verts, dist, pred = _bfs(h, g, [5], False)
    ref_b, _ = oracle.bfs(s, d, V, [5])
    got_b = by_vertex(verts, dist, V)
    assert np.array_equal(got_b, ref_b)
    assert oracle.check_bfs_predecessors(s, d, V, got_b, by_vertex(verts, pred, V), [5])


def check_int64_ids_double_weights(monkeypatch, knobs):
    """int64 vertex ids and float64 weights: PageRank at 1e-9 against the fp64 oracle, SSSP bit-exact"""
    rng = np.random.default_rng(5)
    V, E = 3000, 40000
    ids = rng.choice(np.arange(10**12, 10**12 + 10**7), size=V, replace=False).astype(np.int64)
    s = rng.integers(0, V, E)
    d = rng.integers(0, V, E)
    w = rng.random(E) + 0.5
    for st in (True, False):
        h, g = _graph(monkeypatch, knobs, ids[s], ids[d], w, store_transposed=st, vertex_dtype=np.int64,
                      weight_dtype=np.float64, vertices=ids)
        verts, vals, _ = _pagerank(h, g, 0.85, 0.0, 40)
        assert str(verts.dtype) == "torch.int64" and str(vals.dtype) == "torch.float64"
        ref, _, _ = oracle.pagerank(s, d, V, w, alpha=0.85, epsilon=0.0, max_iterations=40)
        pos = np.searchsorted(np.sort(ids), verts.cpu().numpy())
        got = np.zeros(V)
        got[np.argsort(ids)[pos]] = vals.cpu().numpy()
        np.testing.assert_allclose(got, ref, rtol=1e-9)
        verts, dist, pred = _sssp(h, g, int(ids[3]))
        ref_d, _ = oracle.sssp(s, d, w, V, 3, use_float=False)
        idx = np.argsort(ids)[np.searchsorted(np.sort(ids), verts.cpu().numpy())]
        got_d = np.zeros(V)
        got_d[idx] = dist.cpu().numpy()
        assert np.array_equal(got_d, ref_d)
        p = pred.cpu().numpy()
        got_p = np.full(V, -1, dtype=np.int64)
        got_p[idx[p >= 0]] = np.argsort(ids)[np.searchsorted(np.sort(ids), p[p >= 0])]
        assert oracle.check_sssp_predecessors(s, d, w, V, got_d, got_p, 3)


# =========================================================================================================== tests
def test_offs64_bfs(monkeypatch):
    check_bfs(monkeypatch, OFFS64, 16)


def test_offs64_sssp(monkeypatch):
    check_sssp(monkeypatch, OFFS64, 16)


@pytest.mark.parametrize("wdtype", [np.float32, np.float64])
def test_offs64_sssp_zero_weight_predecessors(monkeypatch, wdtype):
    check_sssp_zero_weights(monkeypatch, OFFS64, wdtype)


@pytest.mark.parametrize("store_transposed,weighted", [(True, False), (True, True), (False, False)])
def test_offs64_pagerank_plain_sweep(monkeypatch, store_transposed, weighted):
    check_pagerank_offs64(monkeypatch, 16, store_transposed, weighted)


def test_offs64_katz_hits_eigenvector(monkeypatch):
    check_siblings(monkeypatch, OFFS64, 14)


def test_offs64_wcc_degrees_extract_paths(monkeypatch):
    check_structure(monkeypatch, OFFS64, 14)


def test_offs64_csr_input(monkeypatch):
    check_csr_input(monkeypatch, OFFS64)


def test_offs64_int64_ids_double_weights(monkeypatch):
    check_int64_ids_double_weights(monkeypatch, OFFS64)


def test_offs64_advance_in_halves(monkeypatch):
    """64-bit offsets with frontiers of 2048 edges or more advanced in halves: the path of a graph with 2^31 edges"""
    knobs = {**OFFS64, "ADVANCE_SPLIT_EDGES": "2048"}
    check_bfs(monkeypatch, knobs, 16, depth_limit=False)
    check_sssp(monkeypatch, knobs, 16, cutoff=False, no_pred=False)


STREAM = {"forced": {"SWEEP_MIN_EDGES": "0"},
          "bands-and-tail": {"SWEEP_MIN_EDGES": "0", "SWEEP_BANDS": "3", "SWEEP_TAIL_DEGREE": "8"}}


@pytest.mark.parametrize("stream", list(STREAM))
@pytest.mark.parametrize("weighted", [False, True])
def test_piece_stream_pagerank_csr(monkeypatch, stream, weighted):
    check_pagerank_stream(monkeypatch, STREAM[stream], 16, weighted)


@pytest.mark.parametrize("stream", list(STREAM))
def test_piece_stream_katz_hits_eigenvector(monkeypatch, stream):
    check_siblings(monkeypatch, STREAM[stream], 15)


SSSP_SCHEDULES = {"not-adaptive": {"SSSP_ADAPTIVE": "0"},
                  "no-single-cta-rounds": {"SSSP_SMALL_ROUNDS": "0"},
                  "split-every-round": {"SSSP_SPLIT_MIN_EDGES": "0", "SSSP_SPLIT_ROUNDS": "1"},
                  "split-every-round-twice": {"SSSP_SPLIT_MIN_EDGES": "0", "SSSP_SPLIT_ROUNDS": "2"},
                  "delta-1/64": {"SSSP_DELTA_SCALE": "0.015625"},
                  "delta-64": {"SSSP_DELTA_SCALE": "64"}}


@pytest.mark.parametrize("schedule", list(SSSP_SCHEDULES))
def test_sssp_schedule(monkeypatch, schedule):
    check_sssp(monkeypatch, SSSP_SCHEDULES[schedule], 16, cutoff=False, no_pred=False)


BFS_SCHEDULES = {"bottom-up-from-the-first-level": {"BFS_ALPHA": "1e9", "BFS_BETA": "1e9"},
                 "never-bottom-up": {"BFS_ALPHA": "0"}}


@pytest.mark.parametrize("schedule", list(BFS_SCHEDULES))
def test_bfs_schedule(monkeypatch, schedule):
    check_bfs(monkeypatch, BFS_SCHEDULES[schedule], 16, directions=(True,), depth_limit=False)
