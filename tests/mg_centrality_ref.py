"""Multi-GPU Katz, eigenvector centrality and HITS on every rank of a grid in ONE process (tests/mg_world.py:
MGGraph.katz_centrality / .eigenvector_centrality / .hits themselves), the single-GPU reference, the graphs and the
checks' helpers.

Shared by tests/test_mg_centrality_cpu.py and tests/test_mg_centrality_gpu.py; the multi-GPU PageRank tests use its graphs."""
import numpy as np

from tests import mg_world


def _worker(rank, world, s, d, w, dtype, device, runs):
    from cugraph_b200 import _capi
    g = mg_world.graph(rank, world, s, d, w, dtype, device)
    out = []
    for algo, kw in runs:
        try:
            if algo == "katz":
                out.append((*g.katz_centrality(**kw), g.last_katz_stats))
            elif algo == "eigenvector":
                out.append((*g.eigenvector_centrality(**kw), g.last_eigenvector_stats))
            else:   # the initial hubs' (ids, values) spread over the ranks
                guess = kw.get("initial_hubs_guess")
                kw = dict(kw, initial_hubs_guess=None if guess is None else mg_world.share(rank, world, *guess))
                out.append((*g.hits(**kw), g.last_hits_stats))
        except _capi.CugraphError as e:
            out.append(str(e))
    return out, g.num_edges_local


def mg_centrality(s, d, V, world, runs, w=None, dtype=np.float32, device="cpu"):
    """runs = [(algorithm "katz" / "eigenvector" / "hits", keywords of its MGGraph method)] on `world` ranks, one graph for
    all runs.  Returns (per run: (values by vertex id, ..., last stats) or the error message every rank raised, the
    number of ranks whose block has no edges)"""
    res = mg_world.run(world, _worker, s, d, w, dtype, device, runs)
    out = []
    for k in range(len(runs)):
        first = res[0][0][k]
        if isinstance(first, str):
            assert all(r[0][k] == first for r in res), k
            out.append(first)
            continue
        assert all(r[0][k][-1] == first[-1] for r in res), k      # every rank ran the same iterations
        out.append(tuple(mg_world.by_id([(r[0][k][0], r[0][k][j]) for r in res], V) for j in range(1, len(first) - 1))
                   + (first[-1],))
    return out, sum(r[1] == 0 for r in res)


def single_gpu(algo, s, d, V, w=None, **kw):
    """cugraph_katz_centrality / _eigenvector_centrality / cugraph_hits on the graph with every id 0..V-1 a vertex, by
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
