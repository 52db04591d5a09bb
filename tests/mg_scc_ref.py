"""Multi-GPU strongly connected components on every rank of a grid in ONE process (tests/mg_world.py:
MGGraph.strongly_connected_components itself), the single-GPU result, the graphs and the checks.

Shared by tests/test_mg_scc_cpu.py and tests/test_mg_scc_gpu.py."""
import json
import os

import numpy as np
import torch

from tests import mg_world
from tests.scc_ref import scc as tarjan

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _graph(rank, world, s, d, w, device, kw):
    """rank's MGGraph from its share of the edge list, with the constructor's keyword options (`vertices` are given by
    rank 0 alone)"""
    from cugraph_b200 import mg
    s, d, *rest = mg_world.share(rank, world, s, d, *([] if w is None else [w]))
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(device)  # noqa: E731
    kw = dict(kw)
    if "vertices" in kw:
        kw["vertices"] = t(kw["vertices"]) if rank == 0 else None
    return mg.MGGraph(t(s), t(d), t(rest[0]) if rest else None,
                      dtype=torch.float64 if w is not None and w.dtype == np.float64 else torch.float32, **kw)


def _worker(rank, world, s, d, w, device, kw, with_wcc):
    g = _graph(rank, world, s, d, w, device, kw)
    v, labels = g.strongly_connected_components()
    assert labels.dtype == v.dtype
    wcc = g.weakly_connected_components()[1] if with_wcc else None
    return v, labels, g.last_scc_stats, g.num_edges_local, wcc


def mg_scc(s, d, V, world, w=None, device="cpu", with_wcc=False, **kw):
    """MGGraph.strongly_connected_components on `world` ranks.  Returns (labels [V] int64: the vertex id each vertex's
    label names, last_scc_stats, the number of ranks whose block has no edges[, MG WCC's labels of the same graph, by id])
    indexed by vertex id; ids that are not vertices of the graph are components of their own"""
    res = mg_world.run(world, _worker, s, d, w, device, kw, with_wcc)
    labels = mg_world.by_id([r[:2] for r in res], V, -1, np.int64)
    absent = labels < 0
    labels[absent] = np.flatnonzero(absent)
    stats = res[0][2]
    assert all(r[2] == stats for r in res)                        # every rank ran the same rounds
    out = (labels, stats, sum(r[3] == 0 for r in res))
    if with_wcc:
        wcc = mg_world.by_id([(r[0], r[4]) for r in res], V, -1, np.int64)
        wcc[absent] = np.flatnonzero(absent)
        out += (wcc,)
    return out


def single_gpu_scc(s, d, V):
    """cugraph_strongly_connected_components on the same directed graph (every id 0..V-1 a vertex): labels by vertex id"""
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import by_vertex, make_graph
    h, g = make_graph(s, d, vertices=np.arange(V, dtype=np.int32))
    verts, labels = plc.strongly_connected_components(h, g, None, None, None, None, False)
    return by_vertex(verts, labels, V)


def same_partition(a, b):
    """the labellings a and b (indexed by vertex) split the vertices into the same sets"""
    return len(set(zip(a.tolist(), b.tolist()))) == len(set(a.tolist())) == len(set(b.tolist()))


def check(s, d, V, labels, single=None):
    """the partition of `labels` is Tarjan's, scipy's (connection="strong") and single-GPU SCC's when given; every label
    is a member of its own SCC and carries its own label"""
    import scipy.sparse as sp
    from scipy.sparse.csgraph import connected_components
    s, d = np.asarray(s, np.int64), np.asarray(d, np.int64)
    ref = tarjan(s, d, V)
    assert labels.shape == (V,)
    assert same_partition(labels, ref)
    _, lab = connected_components(sp.coo_matrix((np.ones(s.size), (s, d)), shape=(V, V)).tocsr(), directed=True,
                                  connection="strong")
    assert same_partition(labels, lab)
    if single is not None:
        assert same_partition(labels, single)
    assert ((labels >= 0) & (labels < V)).all()
    assert np.array_equal(ref[labels], ref)
    assert np.array_equal(labels[labels], labels)


# ---------------------------------------------------------------------------------------------------------- graphs
def golden_cases():
    """the SCC golden fixture: name -> (src, dst, V)"""
    with open(os.path.join(ROOT, "tests", "golden", "scc_golden.json")) as f:
        cases = json.load(f)["cases"]
    out = {}
    for name, c in cases.items():
        s, d = np.asarray(c["src"], np.int32), np.asarray(c["dst"], np.int32)
        out[name] = (s, d, int(c.get("num_vertices") or max(s.max(), d.max()) + 1))
    return out


def c_test_graph():
    """the graph of the reference's multi-GPU SCC C test: (src, dst, V)"""
    with open(os.path.join(ROOT, "tests", "golden", "mg_scc_c_test_graph.json")) as f:
        c = json.load(f)
    return np.asarray(c["src"], np.int32), np.asarray(c["dst"], np.int32), int(c["num_vertices"])


def rmat_graph(scale, seed=900):
    """directed RMAT, ef 16, as generated (multi-edges and self-loops kept)"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed + scale)
    return np.asarray(s, np.int32), np.asarray(d, np.int32), 1 << scale


def _scattered(s, d, V, seed):
    p = np.random.default_rng(seed).permutation(V)
    return p[s].astype(np.int32), p[d].astype(np.int32), V


def chain(n):
    """a directed path of n vertices: the trim peels one vertex from each end per round"""
    return _scattered(np.arange(n - 1), np.arange(1, n), n, n)


def cycle(n):
    """one directed cycle: resolved by the forward-backward step"""
    return _scattered(np.arange(n), (np.arange(n) + 1) % n, n, n + 1)


def cycle_chain(n_cycles, k):
    """n_cycles directed cycles of k vertices, cycle i joined to cycle i + 1 by one edge: colouring rounds"""
    base = np.arange(n_cycles)[:, None] * k
    ring = np.arange(k)
    s = np.concatenate([(base + ring).ravel(), base[:-1, 0] + k // 2])
    d = np.concatenate([(base + (ring + 1) % k).ravel(), base[1:, 0]])
    return _scattered(s, d, n_cycles * k, k)


def split_graph():
    """a complete digraph on 6 vertices (the pivot's SCC) with a 2-cycle X it reaches, a 2-cycle Y that reaches it and a
    2-cycle Z apart: FW\\BW = X and BW\\FW = Y are both non-empty, and the colouring resolves X, Y and Z in one round"""
    k = np.arange(6)
    s, d = np.repeat(k, 6), np.tile(k, 6)
    keep = s != d
    s, d = list(s[keep]), list(d[keep])
    s += [6, 7, 0, 8, 9, 8, 10, 11]                 # X = {6, 7}, 0 -> 6; Y = {8, 9}, 8 -> 1; Z = {10, 11}
    d += [7, 6, 6, 9, 8, 1, 11, 10]
    return _scattered(np.array(s), np.array(d), 12, 3)


def both_directions(n_pairs, V, seed):
    """random edges given in both directions (not declared symmetric)"""
    r = np.random.default_rng(seed)
    a, b = r.integers(0, V, n_pairs), r.integers(0, V, n_pairs)
    return np.concatenate([a, b]).astype(np.int32), np.concatenate([b, a]).astype(np.int32), V


def loops_and_multi_edges(V, E, seed):
    """a random directed graph with a self-loop on a quarter of its vertices and a third of its edges repeated"""
    r = np.random.default_rng(seed)
    s, d = r.integers(0, V, E), r.integers(0, V, E)
    loops = r.choice(V, size=V // 4, replace=False)
    dup = r.integers(0, E, E // 3)
    return (np.concatenate([s, loops, s[dup]]).astype(np.int32), np.concatenate([d, loops, d[dup]]).astype(np.int32), V)


# ---------------------------------------------------------------------------------------------------------- checks
def check_grid(world, device, rmat_scales, big_goldens=True):
    """the golden cases, the reference's MG C-test graph and directed RMAT graphs on one grid"""
    for name, (s, d, V) in golden_cases().items():
        if big_goldens or s.size < 10_000:
            labels, _, _ = mg_scc(s, d, V, world, device=device)
            check(s, d, V, labels, single=single_gpu_scc(s, d, V))
    s, d, V = c_test_graph()
    labels, _, _ = mg_scc(s, d, V, world, device=device)
    check(s, d, V, labels, single=single_gpu_scc(s, d, V))
    assert np.array_equal(labels, np.arange(V))                   # Tarjan: the graph is acyclic, 12 singletons
    for scale in rmat_scales:
        s, d, V = rmat_graph(scale)
        labels, _, _ = mg_scc(s, d, V, world, device=device)
        check(s, d, V, labels, single=single_gpu_scc(s, d, V))


def check_phases(world, device, n, n_cycles, k):
    """one graph per phase, with the rounds that show the phase did the work"""
    s, d, V = chain(n)
    labels, st, _ = mg_scc(s, d, V, world, device=device)
    check(s, d, V, labels)
    assert st["trim_rounds"] == n // 2 and st["fw_rounds"] == 0 and st["outer_rounds"] == 0, st
    s, d, V = cycle(n)
    labels, st, _ = mg_scc(s, d, V, world, device=device)
    check(s, d, V, labels)
    assert st["trim_rounds"] == 0 and st["fw_rounds"] == n and st["bw_rounds"] == n and st["outer_rounds"] == 0, st
    s, d, V = cycle_chain(n_cycles, k)
    labels, st, _ = mg_scc(s, d, V, world, device=device)
    check(s, d, V, labels)
    assert st["outer_rounds"] >= 2 and st["colour_rounds"] > st["outer_rounds"], st
    s, d, V = split_graph()
    labels, st, _ = mg_scc(s, d, V, world, device=device)
    check(s, d, V, labels)
    assert st["trim_rounds"] == 0 and st["fw_rounds"] >= 2 and st["bw_rounds"] >= 2 and st["outer_rounds"] == 1, st


def check_edge_cases(world, device, n_pairs, V, seed):
    """both directions of every edge (= MG WCC's labels), symmetrize=True rejected on every rank, listed isolated vertices,
    self-loops and multi-edges"""
    from cugraph_b200 import _capi
    s, d, V = both_directions(n_pairs, V, seed)
    labels, _, _, wcc = mg_scc(s, d, V, world, device=device, with_wcc=True)
    check(s, d, V, labels)
    assert np.array_equal(labels, wcc)
    for e in mg_world.run(world, _symmetrized_worker, s[:n_pairs], d[:n_pairs], device):
        assert isinstance(e, _capi.CugraphRuntimeError) and e.code == _capi.UNKNOWN_ERROR, e
        assert "Invalid input argument: call weakly_connected_components instead for symmetric graphs." in str(e)
    s, d, V = cycle_chain(6, 3)
    extra = np.arange(V, V + 7, dtype=np.int32)                   # vertices of no edge: singletons
    labels, st, _ = mg_scc(s, d, V + 7, world, device=device, vertices=np.concatenate([extra, s[:5]]))
    check(s, d, V + 7, labels)
    assert np.array_equal(labels[V:], extra)
    s, d, V = loops_and_multi_edges(V * 40, V * 80, seed)
    labels, _, _ = mg_scc(s, d, V, world, device=device)
    check(s, d, V, labels, single=single_gpu_scc(s, d, V))


def _symmetrized_worker(rank, world, s, d, device):
    """the error MGGraph.strongly_connected_components raises on this rank for a graph built with symmetrize=True"""
    g = _graph(rank, world, s, d, None, device, dict(symmetrize=True))
    try:
        g.strongly_connected_components()
    except Exception as e:  # noqa: BLE001  (checked by the caller)
        return e
    return None


def check_empty_blocks(device):
    """a few edges over a 4 x 2 grid: most blocks have none"""
    s = np.array([0, 1, 5, 9, 9, 2, 11], np.int32)
    d = np.array([1, 0, 9, 5, 2, 9, 11], np.int32)
    V = 12
    labels, _, empty = mg_scc(s, d, V, 8, device=device)
    assert empty > 0
    check(s, d, V, labels, single=single_gpu_scc(s, d, V))


def check_weighted(world, device, s, d, V):
    """weighted float32 / float64 blocks give the labels of the unweighted one"""
    want, _, _ = mg_scc(s, d, V, world, device=device)
    for wdtype in (np.float32, np.float64):
        w = np.random.default_rng(1).random(s.size).astype(wdtype)
        got, _, _ = mg_scc(s, d, V, world, w=w, device=device)
        assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------- the entry point
def _block(L, handle, rows, cols, n_rows, n_cols, device):
    import ctypes as C
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View
    keep = [torch.as_tensor(rows, dtype=torch.int32).to(device), torch.as_tensor(cols, dtype=torch.int32).to(device)]
    views = [View(k) for k in keep]
    blk, err = C.c_void_p(), C.c_void_p()
    code = L.cugraph_b200_block_create(handle.ptr, n_rows, n_cols, views[0].ptr, views[1].ptr, None, C.byref(blk),
                                       C.byref(err))
    _capi.check(code, err, "cugraph_b200_block_create")
    return blk.value, (keep, views)


def scc_push(L, handle, blk, transposed, mode, key_src, val_src, key_dst, grid, out):
    """cugraph_b200_block_scc_push; grid = (maxpart, grid_rows, grid_cols, grid_r, grid_c)"""
    import ctypes as C
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View
    vs = [View(t) for t in (key_src, val_src, key_dst, out)]
    err = C.c_void_p()
    try:
        code = L.cugraph_b200_block_scc_push(handle.ptr, blk, transposed, mode, vs[0].ptr, vs[1].ptr, vs[2].ptr, *grid,
                                             vs[3].ptr, C.byref(err))
    finally:
        for v in vs:
            v.free()
    _capi.check(code, err, "cugraph_b200_block_scc_push")


def check_entry_point(device):
    """cugraph_b200_block_scc_push against numpy: both orientations and modes, every source active, a few and none; key
    mismatches filtered out; self-loops (equal codes of the two ends) skipped; 32- and 64-bit offsets"""
    import os
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    L = _capi.lib()
    rng = np.random.default_rng(4)
    m, R, Cc, gr, gc = 150, 2, 3, 1, 2                            # maxpart, grid shape, grid position
    grid = (m, R, Cc, gr, gc)
    n_rows, n_cols, E = Cc * m, R * m, 6000
    rows = np.concatenate([np.full(300, 3), rng.integers(0, n_rows - 50, E - 300)])   # one row of degree >= 300
    cols = np.concatenate([rng.integers(0, n_cols, 300), (rng.integers(0, n_cols, E - 300) * rng.random(E - 300) ** 2)])
    lid = rng.integers(0, m, 40)                                  # self-loops: column block gr, row block gc, same lid
    rows = np.concatenate([rows, gc * m + lid]).astype(np.int64)
    cols = np.concatenate([cols, gr * m + lid]).astype(np.int64)
    col_code = ((cols // m) * Cc + gc) * m + cols % m
    row_code = (gr * Cc + rows // m) * m + rows % m
    assert (col_code == row_code).sum() >= 40
    imin = np.iinfo(np.int64).min

    def model(transposed, mode, key_src, val_src, key_dst):
        src, dst = (rows, cols) if transposed else (cols, rows)
        live = (col_code != row_code) & (val_src[src] != imin) & (key_src[src] == key_dst[dst])
        if mode == 0:
            out = np.full(n_cols if transposed else n_rows, imin, dtype=np.int64)
            np.maximum.at(out, dst[live], val_src[src[live]])
        else:
            out = np.zeros(n_cols if transposed else n_rows, dtype=np.int64)
            np.add.at(out, dst[live], 1)
        return out

    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)  # noqa: E731
    for offs64 in (False, True):
        if offs64:   # read when the handle is created
            os.environ["CUGRAPH_B200_OFFS64_MIN_EDGES"] = "0"
        try:
            handle = ResourceHandle(stream=0)
            blk, keep = _block(L, handle, rows, cols, n_rows, n_cols, device)
        finally:
            os.environ.pop("CUGRAPH_B200_OFFS64_MIN_EDGES", None)
        for transposed in (0, 1):
            n_src, n_dst = (n_rows, n_cols) if transposed else (n_cols, n_rows)
            src = rows if transposed else cols
            deg = np.bincount(src, minlength=n_src)
            few = np.full(n_src, imin, dtype=np.int64)
            act = np.flatnonzero(deg == 1)[:3]
            few[act] = rng.integers(-5, 1 << 40, act.size)
            for mode in (0, 1):
                for val in (rng.integers(-(1 << 40), 1 << 40, n_src), few, np.full(n_src, imin, dtype=np.int64)):
                    for key_src, key_dst in ((np.zeros(n_src, np.int64), np.zeros(n_dst, np.int64)),
                                             (rng.integers(0, 3, n_src), rng.integers(0, 3, n_dst))):
                        out = t(np.full(n_dst + 3, 7, dtype=np.int64))
                        scc_push(L, handle, blk, transposed, mode, t(key_src), t(val), t(key_dst), grid, out)
                        want = model(transposed, mode, key_src, val, key_dst)
                        assert np.array_equal(out.cpu().numpy()[:n_dst], want), (offs64, transposed, mode)
                        assert (out.cpu().numpy()[n_dst:] == 7).all()
                if mode == 1:   # all active: the counts are the live degrees, self-loops left out
                    assert np.array_equal(model(transposed, 1, np.zeros(n_src, np.int64), np.zeros(n_src, np.int64),
                                                np.zeros(n_dst, np.int64)),
                                          np.bincount((cols if transposed else rows)[col_code != row_code],
                                                      minlength=n_dst))
        L.cugraph_b200_block_free(blk)


def check_entry_errors(device):
    """every bad argument returns CUGRAPH_INVALID_INPUT"""
    import ctypes as C
    import pytest
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    handle = ResourceHandle(stream=0)
    blk, keep = _block(L, handle, [0, 1, 2], [1, 2, 0], 3, 4, device)
    i64 = lambda n: torch.zeros(n, dtype=torch.int64).to(device)  # noqa: E731
    good = dict(transposed=0, mode=0, key_src=i64(4), val_src=i64(4), key_dst=i64(3), grid=(2, 2, 2, 0, 0), out=i64(3))

    def call(**kw):
        a = dict(good)
        a.update(kw)
        scc_push(L, handle, blk, a["transposed"], a["mode"], a["key_src"], a["val_src"], a["key_dst"], a["grid"], a["out"])

    call()
    call(transposed=1, key_src=i64(3), val_src=i64(3), key_dst=i64(4), out=i64(4))
    bad = [dict(key_src=i64(4).int()), dict(val_src=i64(4).double()), dict(key_dst=i64(3).int()), dict(out=i64(3).float()),
           dict(key_src=i64(3)), dict(val_src=i64(3)), dict(key_dst=i64(2)), dict(out=i64(2)),
           dict(transposed=1), dict(mode=2), dict(mode=-1),
           dict(grid=(0, 2, 2, 0, 0)), dict(grid=(2, 0, 2, 0, 0)), dict(grid=(2, 2, 0, 0, 0)), dict(grid=(2, 2, 2, 2, 0)),
           dict(grid=(2, 2, 2, -1, 0)), dict(grid=(2, 2, 2, 0, 2)), dict(grid=(2, 2, 2, 0, -1))]
    for kw in bad:
        with pytest.raises(_capi.CugraphError) as e:
            call(**kw)
        assert e.value.code == _capi.INVALID_INPUT, kw
    vs = [View(good[k]) for k in ("key_src", "val_src", "key_dst", "out")]
    err = C.c_void_p()
    for k in range(5):
        args = [blk] + [v.ptr for v in vs]
        args[k] = None
        code = L.cugraph_b200_block_scc_push(handle.ptr, args[0], 0, 0, args[1], args[2], args[3], *good["grid"], args[4],
                                             C.byref(err))
        with pytest.raises(_capi.CugraphError) as e:
            _capi.check(code, err, "cugraph_b200_block_scc_push")
        assert e.value.code == _capi.INVALID_INPUT
    for v in vs:
        v.free()
    L.cugraph_b200_block_free(blk)
