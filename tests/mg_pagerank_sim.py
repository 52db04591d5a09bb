"""Multi-GPU PageRank with every rank in ONE process (tests/mg_grid.py): the real block pull sweeps
(cugraph_b200_block_sweep) and the real owner steps (cugraph_b200_pagerank_vertex_step / _personalized_vertex_step) in the
iteration of MGGraph.pagerank, with personalization, an initial guess and precomputed out-weights placed on their owners
as MGGraph.pagerank places them.

Shared by tests/test_mg_pagerank_cpu.py and tests/test_mg_pagerank_gpu.py."""
import numpy as np

from tests.mg_grid import Grid  # noqa: F401

F32_TOL = dict(rtol=1e-6, atol=1e-12)
F64_TOL = dict(rtol=1e-9, atol=0.0)


def out_weights(s, V, w=None):
    """the out-weight sums by vertex id"""
    return np.bincount(s, weights=None if w is None else np.asarray(w, np.float64), minlength=V).astype(np.float64)


def pagerank(grid, out_w, alpha=0.85, epsilon=0.0, max_iterations=100, personalization=None, initial_guess=None):
    """Returns (values by vertex id, iterations, converged).  out_w, personalization and initial_guess are dense by vertex id
    (personalization: 0 for the vertices not personalized)."""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    P, mp = grid.P, grid.mp
    n = [int(c) for c in grid.counts]

    def owned(vals):
        out = []
        for p in range(P):
            a = grid.zeros(mp)
            a[:n[p]] = grid.t(np.asarray(vals)[grid.own[p]].astype(T))
            out.append(a)
        return out

    ow = owned(out_w)
    pr = owned(np.full(grid.V, 1.0 / grid.V) if initial_guess is None else initial_guess)
    pers = None if personalization is None else owned(personalization)
    pers_sum = None if personalization is None else float(np.asarray(personalization, T).astype(np.float64).sum())
    x = [grid.zeros(mp) for _ in range(P)]
    y = [grid.zeros(mp) for _ in range(P)]
    tot = [grid.scalars(2) for _ in range(P)]

    def step(first):
        parts = [grid.scalars(2) for _ in range(P)]
        for p in range(P):
            if pers is None:
                grid.call("cugraph_b200_pagerank_vertex_step", y[p], pr[p], ow[p], x[p], n[p], float(alpha), float(grid.V),
                          int(first), tot[p], parts[p])
            else:
                grid.call("cugraph_b200_pagerank_personalized_vertex_step", y[p], pr[p], ow[p], x[p], pers[p], n[p],
                          float(alpha), pers_sum, int(first), tot[p], parts[p])
        diff, _ = grid.all_reduce(parts)
        for p in range(P):
            tot[p].copy_(parts[p])
        return diff

    step(True)
    it = 0
    for _ in range(int(max_iterations)):
        y = grid.spmv(x, alpha)
        diff = step(False)
        it += 1
        if epsilon > 0.0 and diff < epsilon:
            break
    return grid.by_vertex(pr), it, it < max_iterations


def oracle_pagerank(s, d, V, w=None, alpha=0.85, epsilon=0.0, max_iterations=100, personalization=None,
                    initial_guess=None, out_w=None):
    """oracle.pagerank with the dense personalization of pagerank() turned into (ids, values)"""
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
