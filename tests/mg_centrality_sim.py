"""Multi-GPU Katz, eigenvector centrality and HITS with every rank in ONE process (tests/mg_grid.py): the real block sweeps
(cugraph_b200_block_sweep, pull and transposed) and the real owner steps (cugraph_b200_katz_step, _eigenvector_add_step /
_scale_step, _hits_max_step / _scale_step, _vertex_sum / _scale) in the iterations of MGGraph's drivers.

Shared by tests/test_mg_centrality_cpu.py and tests/test_mg_centrality_gpu.py, together with the graphs and checks below."""
import numpy as np

from tests.mg_grid import Grid  # noqa: F401


def katz(grid, alpha, beta=1.0, epsilon=1e-6, max_iterations=100):
    """Returns (values by vertex id, iterations); the iteration of MGGraph.katz_centrality"""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    x = [grid.zeros(grid.mp) for _ in range(grid.P)]
    it = 0
    while True:
        y = grid.spmv(x, alpha)
        parts = [grid.scalars(2) for _ in range(grid.P)]
        for p in range(grid.P):
            grid.call("cugraph_b200_katz_step", y[p], x[p], int(grid.counts[p]), float(beta), parts[p])
        diff, sumsq = grid.all_reduce(parts)
        it += 1
        if T(diff) < T(epsilon):
            break
        if it >= max_iterations:
            raise RuntimeError("Katz Centrality failed to converge.")
    for p in range(grid.P):
        grid.call("cugraph_b200_vertex_scale", x[p], int(grid.counts[p]), 1.0 / float(np.sqrt(sumsq)))
    return grid.by_vertex(x), it


def eigenvector(grid, epsilon=1e-6, max_iterations=100):
    """Returns (values by vertex id, iterations); the iteration of MGGraph.eigenvector_centrality"""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    x = []
    for p in range(grid.P):
        xp = grid.zeros(grid.mp)
        xp[:grid.counts[p]] = 1.0 / grid.V
        x.append(xp)
    it = 0
    while True:
        y = grid.spmv(x, 1.0)
        sq = [grid.scalars(1) for _ in range(grid.P)]
        for p in range(grid.P):
            grid.call("cugraph_b200_eigenvector_add_step", y[p], x[p], int(grid.counts[p]), sq[p])
        grid.all_reduce(sq)
        parts = [grid.scalars(1) for _ in range(grid.P)]
        for p in range(grid.P):
            grid.call("cugraph_b200_eigenvector_scale_step", y[p], x[p], int(grid.counts[p]), sq[p], parts[p])
        diff, = grid.all_reduce(parts)
        it += 1
        if T(diff) < T(grid.V) * T(epsilon):
            break
        if it >= max_iterations:
            raise RuntimeError("Eigenvector Centrality failed to converge.")
    return grid.by_vertex(x), it


def hits(grid, epsilon=1e-5, max_iterations=100, initial_hubs=None, normalize=True):
    """Returns (hubs, authorities by vertex id, iterations, last difference); the iteration of MGGraph.hits.  initial_hubs:
    values by vertex id (already with the owners: MGGraph.hits moves them there with an all-to-all)"""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    P, mp = grid.P, grid.mp
    n = [int(c) for c in grid.counts]

    def l1(vecs):
        parts = [grid.scalars(1) for _ in range(P)]
        for p in range(P):
            grid.call("cugraph_b200_vertex_sum", vecs[p], n[p], 0, parts[p])
        norm, = grid.all_reduce(parts)
        assert T(norm) > 0
        for p in range(P):
            grid.call("cugraph_b200_vertex_scale", vecs[p], n[p], 1.0 / norm)

    prev = []
    for p in range(P):
        h = grid.zeros(mp)
        h[:n[p]] = 1.0 / grid.V if initial_hubs is None else grid.t(np.asarray(initial_hubs)[grid.own[p]].astype(T))
        prev.append(h)
    if initial_hubs is not None:
        l1(prev)
    it, diff = 0, 0.0
    while True:
        auth = grid.spmv(prev, 1.0, use_weights=False)
        curr = grid.spmv(auth, 1.0, transposed=True, use_weights=False)
        mx = [grid.scalars(2) for _ in range(P)]
        for p in range(P):
            grid.call("cugraph_b200_hits_max_step", curr[p], auth[p], n[p], mx[p])
        h_max, a_max = grid.all_reduce(mx, op="max")
        assert h_max > 0 and a_max > 0
        parts = [grid.scalars(1) for _ in range(P)]
        for p in range(P):
            grid.call("cugraph_b200_hits_scale_step", curr[p], auth[p], prev[p], n[p], mx[p], parts[p])
        d, = grid.all_reduce(parts)
        diff = float(T(d))
        prev = curr
        it += 1
        if T(diff) < T(grid.V) * T(epsilon):
            break
        if it >= max_iterations:
            raise RuntimeError("HITS failed to converge.")
    if normalize:
        l1(prev)
        l1(auth)
    return grid.by_vertex(prev), grid.by_vertex(auth), it, diff


# ---------------------------------------------------------------------------------------------------------------------
# single GPU, graphs, checks
# ---------------------------------------------------------------------------------------------------------------------
def single_gpu(algo, s, d, V, w=None, **kw):
    """cugraph_katz_centrality / _eigenvector_centrality / cugraph_hits on the same graph (every id 0..V-1 a vertex), by
    vertex id.  Katz and eigenvector: (values, None); HITS: (hubs, authorities)."""
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import by_vertex, make_graph
    wdt = np.float32 if w is None else w.dtype
    h, g = make_graph(s, d, weights=w, store_transposed=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=wdt)
    if algo == "katz":
        v, x = plc.katz_centrality(h, g, None, kw["alpha"], kw.get("beta", 1.0), kw["epsilon"], kw["max_iterations"], False)
        return by_vertex(v, x, V).astype(np.float64), None
    if algo == "eigenvector":
        v, x = plc.eigenvector_centrality(h, g, kw["epsilon"], kw["max_iterations"], False)
        return by_vertex(v, x, V).astype(np.float64), None
    v, hb, au = plc.hits(h, g, kw["epsilon"], kw["max_iterations"], None, None, True, False)
    return by_vertex(v, hb, V).astype(np.float64), by_vertex(v, au, V).astype(np.float64)


def katz_alpha(d, V):
    """api.katz_centrality's default on a directed graph: 1 / (1 + the largest in-degree)"""
    return 1.0 / (1.0 + float(np.bincount(d, minlength=V).max()))


def rmat_graph(scale, seed=900):
    """directed RMAT, ef 16"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed + scale)
    return np.asarray(s, np.int32), np.asarray(d, np.int32), 1 << scale


def odd_graph(seed=7):
    """directed: a small RMAT, a chain, sources without in-edges, sinks without out-edges, a 2-cycle, duplicate edges and
    isolated ids, with the ids scattered"""
    from oracle.rmat import rmat_edgelist
    rs, rd = rmat_edgelist(6, 8 << 6, seed=seed)
    parts_s, parts_d = [np.asarray(rs, np.int64)], [np.asarray(rd, np.int64)]
    base = 1 << 6
    chain = np.arange(base, base + 20)
    parts_s += [chain[:-1], np.full(10, chain[0])]                 # the chain and a fan out of its head
    parts_d += [chain[1:], np.arange(base + 20, base + 30)]        # the fan's leaves are sinks
    base += 30
    parts_s += [np.arange(base, base + 8), np.array([base + 8, base + 9, base + 8])]   # 8 sources into the RMAT part
    parts_d += [np.arange(8), np.array([base + 9, base + 8, base + 9])]                # a 2-cycle with a duplicate edge
    base += 10
    V = base + 6                                                  # the last six ids are isolated
    s, d = np.concatenate(parts_s), np.concatenate(parts_d)
    perm = np.random.default_rng(seed).permutation(V)
    return perm[s].astype(np.int32), perm[d].astype(np.int32), V


def tiny_graph():
    """five edges over 12 vertices: on a 4x2 grid most blocks have no edges"""
    s = np.array([0, 1, 5, 9, 2], np.int32)
    d = np.array([1, 5, 9, 2, 0], np.int32)
    return s, d, 12
