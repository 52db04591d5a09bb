"""CPU oracle of betweenness centrality: a restatement of the reference's test oracle
(cpp/tests/centrality/betweenness_centrality_reference.hpp: ref_bfs, ref_accumulation, ref_endpoints_accumulation,
ref_edge_accumulation) and of the scale factors of cpp/src/centrality/betweenness_centrality_impl.cuh (vertex :1432-1490,
edge :1581-1606).  Brandes' algorithm by hops over an edge list (weights are never used), level by level with numpy.

Path counts are fp64 by default; exact=True keeps them as Python integers (object arrays), for graphs whose path counts pass
2^53.  Accumulations are fp64.  Multi-edges each count as a path edge, as in the reference's BFS; self-loops never lie on a
shortest path.  Edge values are per edge-list position, so parallel edges each get their own (equal) value."""
import numpy as np


def _csr(src, dst, V):
    order = np.argsort(src, kind="stable")
    off = np.zeros(V + 1, np.int64)
    np.add.at(off, np.asarray(src, np.int64) + 1, 1)
    return np.cumsum(off), np.asarray(dst, np.int64)[order], order


def _positions(off, f):
    """CSR positions of the out-edges of the vertices f, vertex after vertex"""
    lens = off[f + 1] - off[f]
    total = int(lens.sum())
    if total == 0:
        return np.zeros(0, np.int64)
    first = np.repeat(off[f] - (np.cumsum(lens) - lens), lens)
    return first + np.arange(total)


def brandes(src, dst, V, sources, endpoints=False, edges=False, exact=False):
    """(bc [V], ebc [E] or None, per-source sigma list if exact) unscaled, summed over `sources` (duplicates count twice)"""
    src, dst = np.asarray(src, np.int64), np.asarray(dst, np.int64)
    off, nbr, order = _csr(src, dst, V)
    deg = np.diff(off)
    e_src = np.repeat(np.arange(V), deg)  # CSR position -> source vertex
    bc = np.zeros(V)
    ebc = np.zeros(src.size) if edges else None
    sigmas = []
    for s in np.asarray(sources, np.int64).tolist():
        dist = np.full(V, -1, np.int64)
        sigma = np.zeros(V, object) if exact else np.zeros(V)
        dist[s], sigma[s] = 0, 1
        levels = [np.array([s], np.int64)]
        while True:  # ref_bfs: every edge u -> v with dist[v] == dist[u] + 1 adds sigma[u] to sigma[v]
            f = levels[-1]
            pos = _positions(off, f)
            v = nbr[pos]
            new = np.unique(v[dist[v] < 0])
            if new.size == 0:
                break
            dist[new] = len(levels)
            keep = dist[v] == len(levels)
            np.add.at(sigma, v[keep], sigma[e_src[pos[keep]]])
            levels.append(new)
        delta = np.zeros(V)
        for d in range(len(levels) - 1, 0, -1):  # ref_accumulation / ref_edge_accumulation, deepest level first
            f = levels[d - 1]
            pos = _positions(off, f)
            v = nbr[pos]
            keep = dist[v] == d
            pos, v, u = pos[keep], v[keep], e_src[pos[keep]]
            if exact:
                c = np.array([a / b for a, b in zip(sigma[u].tolist(), sigma[v].tolist())], float) * (1.0 + delta[v])
            else:
                c = sigma[u] / sigma[v] * (1.0 + delta[v])
            np.add.at(delta, u, c)
            if edges:
                np.add.at(ebc, order[pos], c)
        reached = dist >= 0
        if endpoints:  # ref_endpoints_accumulation: the source gets reached - 1, every other reached vertex delta + 1
            bc[reached] += delta[reached] + 1.0
            bc[s] += np.count_nonzero(reached) - 1 - (delta[s] + 1.0)
        else:
            delta[s] = 0.0
            bc += delta
        if exact:
            sigmas.append(sigma)
    return bc, ebc, sigmas


def vertex_scales(V, n_sources, normalized, endpoints, symmetric, dtype=np.float32):
    """(scale of a non-source, scale of a source) or None: betweenness_centrality_impl.cuh:1432-1490 in the weight type"""
    T = dtype
    nv = T(V)
    if not endpoints:
        nv = T(nv - T(1))
    ns = T(n_sources)
    with np.errstate(all="ignore"):
        if T(n_sources) == nv or endpoints:
            if normalized:
                s = T(ns * (nv - T(1)))
            elif symmetric:
                s = T(ns * T(2)) / nv
            else:
                s = ns / nv
            return s, s
        if normalized:
            return T(ns * (nv - T(1))), T(T(n_sources - 1) * (nv - T(1)))
        s_non, s_src = T(ns / nv), T(T(n_sources - 1) / nv)
        if symmetric:
            s_non, s_src = T(s_non * T(2)), T(s_src * T(2))
        return s_non, s_src


def betweenness(src, dst, V, sources=None, normalized=True, endpoints=False, symmetric=False, dtype=np.float32, exact=False):
    """the library's vertex result, by vertex id: sources=None is every vertex"""
    srcs = np.arange(V) if sources is None else np.asarray(sources, np.int64)
    bc, _, _ = brandes(src, dst, V, srcs, endpoints=endpoints, exact=exact)
    s_non, s_src = vertex_scales(V, srcs.size, normalized, endpoints, symmetric, dtype)
    is_src = np.zeros(V, bool)
    is_src[srcs] = True
    with np.errstate(all="ignore"):
        return np.where(is_src, bc.astype(dtype) / s_src, bc.astype(dtype) / s_non).astype(dtype)


def edge_betweenness(src, dst, V, sources=None, normalized=True, symmetric=False, dtype=np.float32):
    """the library's edge result, per edge-list position: sources=None is every vertex"""
    srcs = np.arange(V) if sources is None else np.asarray(sources, np.int64)
    _, ebc, _ = brandes(src, dst, V, srcs, edges=True)
    T = dtype
    sf = None
    if normalized:
        sf = T(T(V) * (T(V) - T(1)))
    elif symmetric:
        sf = T(2)
    if sf is None or V <= 1:
        return ebc.astype(dtype)
    if srcs.size < V:
        sf = T(sf * T(T(srcs.size) / T(V)))
    return (ebc.astype(dtype) / sf).astype(dtype)
