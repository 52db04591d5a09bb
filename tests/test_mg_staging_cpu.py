"""MGGraph's construction options on the CPU, over the emulated library (tests/emu_py.py).

- cugraph_b200_block_stage_edges against the numpy restatement (tests/mg_staging_ref.py): duplicates of equal and distinct
  weights, reverse pairs with more copies one way, an empty input, unweighted / float32 / float64; and its error paths.
- Every rank of a 1x2, 2x1, 2x2 and 4x2 grid in one process (tests/mg_world.py) against the single-GPU constructor with the
  same options, on the hand-made graph with isolated vertices passed in three ways and on RMAT-8: degrees (also against
  numpy), SSSP and BFS bit-exact, PageRank, WCC (from one-direction input with symmetrize), Katz, eigenvector, HITS.
- drop_self_loops + drop_multi_edges on an input with neither: the default constructor's vertices and PageRank, bit for bit.
- A `vertices` dtype error on one rank, a rank over the staging size bound and a staging call failing on one rank: every
  rank raises.
- World sizes 2 and 4 over gloo (the real process groups) against the numpy restatement and the oracle."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_staging_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]
CENTRALITY = [("katz", dict(alpha=0.05, epsilon=1e-7, max_iterations=1000)),
              ("eigenvector", dict(epsilon=1e-7, max_iterations=1000)),
              ("hits", dict(epsilon=1e-7, max_iterations=1000))]


# ---------------------------------------------------------------------------------------------------- the entry point
def _same(got, want):
    assert len(got) == len(want)
    for a, b in zip(got, want):
        assert a[:2] == b[:2]
        assert np.asarray(a[2]).tobytes() == np.asarray(b[2], dtype=np.asarray(a[2]).dtype).tobytes(), (a, b)


@pytest.mark.parametrize("wdtype", [None, np.float32, np.float64], ids=["unweighted", "f32", "f64"])
def test_block_stage_edges_against_numpy_emulated(surface, wdtype):
    rng = np.random.default_rng(11)
    for dm in (False, True):
        for sym in (False, True):
            for n_rows, n_cols, n in ((50, 70, 3000), (3, 2, 40), (1000, 9, 500)):
                rows, cols, rev, w = refs.random_block(rng, n_rows, n_cols, n, wdtype)
                _same(refs.stage_block(rows, cols, rev, w, n_rows, n_cols, dm, sym),
                      refs.stage_block_np(rows, cols, rev, w, dm, sym))
            empty = np.zeros(0, np.int32)
            assert refs.stage_block(empty, empty, empty.astype(np.uint8), None if wdtype is None else empty.astype(wdtype),
                                    4, 4, dm, sym) == []


def test_block_stage_edges_pairing_emulated(surface):
    """one position: 3 originals and 2 reversed copies -> two averaged edges and the heaviest original; dedupe first"""
    rows = np.array([1, 1, 1, 1, 1], np.int32)
    cols = np.array([2, 2, 2, 2, 2], np.int32)
    rev = np.array([0, 1, 0, 1, 0], np.uint8)
    w = np.array([5.0, 4.0, 1.0, 0.5, 3.0], np.float32)
    assert [e[2] for e in refs.stage_block(rows, cols, rev, w, 3, 3, False, True)] == [0.75, 3.5, 5.0]
    assert [e[2] for e in refs.stage_block(rows, cols, rev, w, 3, 3, True, True)] == [0.75]
    assert [e[2] for e in refs.stage_block(rows, cols, rev, w, 3, 3, True, False)] == [0.5]


def test_block_stage_edges_errors_emulated(surface):
    from cugraph_b200 import _capi
    rows = np.array([0, 1, 2], np.int32)
    cols = np.array([1, 2, 0], np.int32)
    rev = np.array([0, 1, 0], np.uint8)
    w = np.array([0.5, 0.25, 1.0], np.float32)
    bad = [dict(rows=rows[:2]), dict(rows=rows.astype(np.int64)), dict(cols=cols.astype(np.int64)),
           dict(w=w[:2]), dict(w=w.astype(np.int32)), dict(rev=rev[:2]), dict(rev=rev.astype(np.int32)),
           dict(n_rows=2), dict(n_cols=2), dict(rows=np.array([0, -1, 2], np.int32)), dict(cols=np.array([1, 2, -3], np.int32)),
           dict(n_rows=1 << 31)]
    for kw in bad:
        args = dict(rows=rows, cols=cols, rev=rev, w=w, n_rows=3, n_cols=3)
        args.update(kw)
        with pytest.raises(_capi.CugraphError) as e:
            refs.stage_block(args["rows"], args["cols"], args["rev"], args["w"], args["n_rows"], args["n_cols"], True, True)
        assert e.value.code == _capi.INVALID_INPUT, kw
    assert len(refs.stage_block(rows, cols, rev, w, 3, 3, True, True)) == 3


# ---------------------------------------------------------------------------------------------------- MG vs single GPU
def _runs(weighted, sources):
    runs = [("pagerank", dict(alpha=0.85, epsilon=0.0, max_iterations=30))]
    runs += [("bfs", dict(source=int(x))) for x in sources]
    if weighted:
        runs += [("sssp", dict(source=int(x))) for x in sources]
    return runs


def _check(s, d, w, world, opts, vertex_lists, runs, device="cpu", partition=()):
    ids = None if vertex_lists is None else np.unique(np.concatenate([v for v in vertex_lists if v is not None]))
    mg = refs.mg_run(s, d, w, world, opts, runs, vertex_lists, device)
    sg = refs.single_gpu(s, d, w, ids, opts, runs)
    verts, (S, D, _) = refs.stage_graph_np(s, d, w, ids, **opts)
    din, dout = refs.degrees_np(verts, S, D)
    assert sorted(mg["in"]) == verts.tolist()
    assert [mg["in"][v] for v in verts.tolist()] == din.tolist()
    assert [mg["out"][v] for v in verts.tolist()] == dout.tolist()
    refs.compare(mg, sg, exact=("bfs", "sssp"), rel=dict(pagerank=1e-6, katz=1e-5, eigenvector=1e-5, hits=1e-5,
                                                          hits_auth=1e-5), partition=partition)
    return mg


@pytest.mark.parametrize("opts", refs.OPTIONS, ids=refs.OPTION_IDS)
@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_staging_hand_graph_emulated(surface, monkeypatch, R, Cc, opts):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, w, iso = refs.hand_graph()
    runs = _runs(True, [0, 8, 40]) + [("wcc", {})] * opts["symmetrize"]
    for wdtype in (np.float32, np.float64):
        for split in refs.vertex_splits(iso, s, world):
            mg = _check(s, d, w.astype(wdtype), world, opts, split, runs, partition=("wcc",))
            assert mg[("sssp", "{'source': 40}")][41] == np.finfo(wdtype).max
    _check(s, d, None, world, opts, [iso] + [None] * (world - 1), _runs(False, [2]) + CENTRALITY)


@pytest.mark.parametrize("opts", refs.OPTIONS, ids=refs.OPTION_IDS)
@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_staging_rmat_emulated(surface, monkeypatch, R, Cc, opts):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, w, V = refs.rmat_graph(8)
    extra = np.arange(V, V + 6, dtype=np.int32)
    runs = _runs(True, [int(s[0]), int(d[7])]) + [("wcc", {})] * opts["symmetrize"]
    _check(s, d, w, world, opts, [extra[:4]] + [None] * (world - 2) + [extra[2:]], runs, partition=("wcc",))


def test_mg_symmetrize_wcc_one_direction_emulated(surface, monkeypatch):
    """WCC from one-direction input: symmetrize=True gives single GPU's partition; isolated ids are singletons"""
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, w, iso = refs.hand_graph()
    mg = _check(s, d, None, world, dict(symmetrize=True), [None, iso, None, None], [("wcc", {})], partition=("wcc",))
    labels = mg[("wcc", "")]
    assert all(labels[v] == v for v in iso)
    assert labels[8] == labels[9] == labels[10] != labels[5]


# ---------------------------------------------------------------------------------------------------- no-op staging
def _noop_worker(rank, world, s, d, w, opts):
    import torch
    from cugraph_b200 import mg
    s_, d_, w_ = mg_world.share(rank, world, s, d, w)
    g = mg.MGGraph(torch.as_tensor(s_), torch.as_tensor(d_), torch.as_tensor(w_), **opts)
    v, x, _, _ = g.pagerank(epsilon=0.0, max_iterations=20)
    return v.numpy(), x.numpy()


@pytest.mark.parametrize("R,Cc", [(2, 2), (4, 2)], ids=["2x2", "4x2"])
def test_mg_noop_staging_bit_identical_emulated(surface, monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, w, V = refs.rmat_graph(8)
    key = s.astype(np.int64) * V + d
    first = np.unique(key, return_index=True)[1]
    keep = np.sort(first[s[first] != d[first]])
    s, d, w = s[keep], d[keep], w[keep]
    plain = mg_world.run(world, _noop_worker, s, d, w, {})
    staged = mg_world.run(world, _noop_worker, s, d, w, dict(drop_self_loops=True, drop_multi_edges=True))
    for (v0, x0), (v1, x1) in zip(plain, staged):
        assert np.array_equal(v0, v1)
        assert x0.tobytes() == x1.tobytes()


# ---------------------------------------------------------------------------------------------------- errors
def _error_worker(rank, world, s, d):
    import torch
    from cugraph_b200 import mg
    s_, d_ = mg_world.share(rank, world, s, d)
    vertices = torch.tensor([100, 101], dtype=torch.int64 if rank == world - 1 else torch.int32)
    try:
        mg.MGGraph(torch.as_tensor(s_), torch.as_tensor(d_), vertices=vertices, symmetrize=True)
    except TypeError as e:
        return str(e)
    return None


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 2)], ids=["1x2", "2x2"])
def test_mg_vertices_dtype_error_on_every_rank_emulated(surface, monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, _, _ = refs.hand_graph()
    got = mg_world.run(world, _error_worker, s, d)
    assert got[0] is not None and "vertices" in got[0]
    assert all(g == got[0] for g in got)


def _raise_worker(rank, world, s, d, w, opts):
    import torch
    from cugraph_b200 import mg
    s_, d_, w_ = mg_world.share(rank, world, s, d, w)
    try:
        mg.MGGraph(torch.as_tensor(s_), torch.as_tensor(d_), torch.as_tensor(w_), **opts)
    except Exception as e:  # noqa: BLE001
        return type(e).__name__, str(e)
    return None


def test_mg_staging_size_bound_on_every_rank_emulated(surface, monkeypatch):
    """a rank with more shuffled edges than staging takes: the same ValueError on every rank, before any staging call"""
    from cugraph_b200 import mg
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, w, _ = refs.hand_graph()
    for opts, name in ((dict(symmetrize=True), "STAGE_MAX_SYMMETRIZED"), (dict(drop_multi_edges=True), "STAGE_MAX_WEIGHTED")):
        monkeypatch.setattr(mg, name, 4)
        got = mg_world.run(world, _raise_worker, s, d, w, opts)
        assert got[0] is not None and got[0][0] == "ValueError" and "too many edges" in got[0][1]
        assert all(g == got[0] for g in got)
        monkeypatch.undo()
        world = mg_world.grid_world(monkeypatch, 2, 2)


def test_mg_staging_failure_on_one_rank_raises_everywhere_emulated(surface, monkeypatch):
    """cugraph_b200_block_stage_edges failing on one rank only (e.g. out of memory there): every rank raises, none goes on
    into the block build and the collectives after it"""
    from cugraph_b200 import _capi, mg
    world = mg_world.grid_world(monkeypatch, 2, 2)
    real = mg.MGGraph._call

    def failing(self, name, *args):
        if name == "cugraph_b200_block_stage_edges" and mg.dist.get_rank() == 2:
            raise _capi.CugraphRuntimeError(_capi.ALLOC_ERROR, "out of memory", name)
        return real(self, name, *args)

    monkeypatch.setattr(mg.MGGraph, "_call", failing)
    s, d, w, _ = refs.hand_graph()
    got = mg_world.run(world, _raise_worker, s, d, w, dict(symmetrize=True))
    assert all(g is not None and g[0] == "CugraphRuntimeError" for g in got)
    assert "out of memory" in got[2][1]
    assert all("failed on another rank" in g[1] for k, g in enumerate(got) if k != 2)


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_worker(rank, world, opts):
    import torch
    from cugraph_b200 import mg
    s, d, w, iso = refs.hand_graph()
    s_, d_, w_ = mg_world.share(rank, world, s.astype(np.int64), d.astype(np.int64), w)
    g = mg.MGGraph(torch.from_numpy(s_), torch.from_numpy(d_), torch.from_numpy(w_),
                   vertices=torch.from_numpy(iso.astype(np.int64)) if rank == world - 1 else None, **opts)
    v, din, dout = mg.degrees(g)
    _, dist, _ = mg.sssp(g, 0, compute_predecessors=False)
    _, labels = mg.weakly_connected_components(g)
    return v.numpy(), din.numpy(), dout.numpy(), dist.numpy(), labels.numpy()


@pytest.mark.parametrize("world", [2, 4])
def test_mg_staging_emulated_gloo(world):
    import oracle
    s, d, w, iso = refs.hand_graph()
    opts = dict(drop_self_loops=True, drop_multi_edges=True, symmetrize=True)
    res = mg_procs.run(_gloo_worker, world, opts, emulated=True)
    verts, (S, D, W) = refs.stage_graph_np(s, d, w, iso, **opts)
    din, dout = refs.degrees_np(verts, S, D)
    V = int(verts.max()) + 1
    want_dist, _ = oracle.sssp(S, D, W, V, 0, cutoff=None, use_float=False)
    want_cc = oracle.wcc(S, D, V)
    got = {}
    for v, a, b, x, lab in res:
        for k in range(v.size):
            got[int(v[k])] = (a[k], b[k], x[k], lab[k])
    assert sorted(got) == verts.tolist()
    for i, v in enumerate(verts.tolist()):
        a, b, x, lab = got[v]
        assert (a, b) == (din[i], dout[i])
        assert x == (want_dist[v] if want_dist[v] < np.finfo(np.float64).max else np.finfo(np.float64).max)
        assert want_cc[lab] == want_cc[v]
