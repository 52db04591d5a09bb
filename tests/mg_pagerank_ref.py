"""Multi-GPU PageRank on every rank of a grid in ONE process (tests/mg_world.py: MGGraph.pagerank itself, with
personalization, an initial guess and precomputed out-weights through its arguments), the oracle and the personalization
cases.

Shared by tests/test_mg_pagerank_cpu.py and tests/test_mg_pagerank_gpu.py."""
import numpy as np

from tests import mg_world

F32_TOL = dict(rtol=1e-6, atol=1e-12)
F64_TOL = dict(rtol=1e-9, atol=0.0)


def out_weights(s, V, w=None):
    """the out-weight sums by vertex id"""
    return np.bincount(s, weights=None if w is None else np.asarray(w, np.float64), minlength=V).astype(np.float64)


def _worker(rank, world, s, d, w, dtype, device, runs):
    g = mg_world.graph(rank, world, s, d, w, dtype, device)
    out = []
    for kw in runs:   # every (ids, values) pair spread over the ranks
        v, x, it, conv = g.pagerank(**{k: mg_world.share(rank, world, *a) if isinstance(a, tuple) else a
                                       for k, a in kw.items()})
        out.append((v, x, it, conv))
    return out


def mg_pagerank(s, d, V, world, runs, w=None, dtype=np.float32, device="cpu"):
    """MGGraph.pagerank on `world` ranks, one graph for all runs (keyword dicts of MGGraph.pagerank).  Per run: (values
    by vertex id, iterations, converged)"""
    res = mg_world.run(world, _worker, s, d, w, dtype, device, runs)
    out = []
    for k in range(len(runs)):
        it, conv = res[0][k][2:]
        assert all(r[k][2:] == (it, conv) for r in res)           # every rank ran the same iterations
        out.append((mg_world.by_id([r[k][:2] for r in res], V), it, conv))
    return out


def oracle_pagerank(s, d, V, w=None, alpha=0.85, epsilon=0.0, max_iterations=100, personalization=None,
                    initial_guess=None, out_w=None):
    """oracle.pagerank with a dense personalization (by vertex id, 0 = not personalized) turned into (ids, values)"""
    import oracle
    pers = None
    if personalization is not None:
        ids = np.flatnonzero(np.asarray(personalization) != 0).astype(np.int32)
        pers = (ids, np.asarray(personalization, np.float64)[ids])
    return oracle.pagerank(s, d, V, None if w is None else np.asarray(w, np.float64), alpha=alpha, epsilon=epsilon,
                           max_iterations=max_iterations, personalization=pers, initial_guess=initial_guess,
                           precomputed_out_w=out_w)


def special_vertices(s, d, V):
    """(a sink with in-edges, a vertex with out-edges but no in-edges, an id without edges) of the graph, -1 where it has none"""
    outd, ind = np.bincount(s, minlength=V), np.bincount(d, minlength=V)

    def first(mask):
        idx = np.flatnonzero(mask)
        return int(idx[0]) if idx.size else -1
    return first((outd == 0) & (ind > 0)), first((ind == 0) & (outd > 0)), first((ind == 0) & (outd == 0))


def cases(s, d, V, seed=0):
    """personalization vectors (dense by vertex id) of the tests: one vertex, a sink, a vertex without in-edges, an isolated
    id, a random share with zeros among the values"""
    rng = np.random.default_rng(seed)
    sink, source, isolated = special_vertices(s, d, V)
    out = {}
    hub = int(np.bincount(d, minlength=V).argmax())
    for name, v in (("one", hub), ("sink", sink), ("no_in_edges", source), ("isolated", isolated)):
        if v >= 0:
            pv = np.zeros(V)
            pv[v] = 1.0
            out[name] = pv
    pv = np.zeros(V)
    pick = rng.choice(V, size=max(V // 8, 2), replace=False)
    pv[pick] = rng.uniform(0.0, 1.0, pick.size)
    pv[pick[::4]] = 0.0
    out["share_with_zeros"] = pv
    return out
