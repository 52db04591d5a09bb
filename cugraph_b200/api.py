"""User-level Python layer for the hot path, in the shape of the reference's `cugraph` package
(python/cugraph/cugraph/structure/graph_classes.py, link_analysis/pagerank.py, traversal/bfs.py, traversal/sssp.py,
centrality/katz_centrality.py, link_analysis/hits.py, components/connectivity.py): a `Graph` built from an edge-list data frame
and functions that return one row per vertex.  cudf is not part of this image: data frames are pandas (the reference accepts
pandas edge lists through `Graph.from_pandas_edgelist` too), arrays move to the device through torch.  Everything below is
argument plumbing over `cugraph_b200.pylibcugraph`; results come from the CUDA library (no CPU path)."""
from __future__ import annotations

import numpy as np


def _plc():
    from cugraph_b200 import pylibcugraph as plc
    return plc


def _dev(a, dtype=None):
    import torch
    t = torch.as_tensor(np.array(np.asarray(a) if dtype is None else np.asarray(a, dtype=dtype), copy=True, order="C"))
    return t.cuda()


def _host(t):
    return t.cpu().numpy()


class Graph:
    """cugraph.Graph(directed=False) — an undirected graph is symmetrised at creation, as the reference does."""

    def __init__(self, directed: bool = False):
        self.directed = bool(directed)
        self.weighted = False
        self._handle = None
        self._graphs = {}      # store_transposed -> SGGraph (PageRank / Katz / HITS want the transposed storage, traversals the other)
        self._edges = None

    # the reference's name for the cudf variant; here both take a pandas data frame (or anything with column access)
    def from_pandas_edgelist(self, pdf, source="source", destination="destination", edge_attr=None, weight=None, renumber=True,
                             vertices=None):
        w_col = edge_attr if edge_attr is not None else weight
        src = np.asarray(pdf[source])
        dst = np.asarray(pdf[destination])
        if src.dtype != dst.dtype or src.dtype not in (np.int32, np.int64):
            dt = np.int64 if max(src.dtype.itemsize, dst.dtype.itemsize) > 4 else np.int32
            src, dst = src.astype(dt), dst.astype(dt)
        w = None
        if w_col is not None:
            w = np.asarray(pdf[w_col])
            if w.dtype not in (np.float32, np.float64):
                w = w.astype(np.float32)
        self._edges = (src, dst, w, bool(renumber), None if vertices is None else np.asarray(vertices, dtype=src.dtype))
        self.weighted = w is not None
        self._graphs = {}
        return self

    from_cudf_edgelist = from_pandas_edgelist

    def _plc_graph(self, store_transposed: bool):
        plc = _plc()
        if self._edges is None:
            raise RuntimeError("the graph has no edges: call from_pandas_edgelist first")
        if self._handle is None:
            self._handle = plc.ResourceHandle()
        key = bool(store_transposed)
        if key not in self._graphs:
            src, dst, w, renumber, vertices = self._edges
            props = plc.GraphProperties(is_symmetric=not self.directed, is_multigraph=True)
            self._graphs[key] = plc.SGGraph(self._handle, props, _dev(src), _dev(dst), weight_array=None if w is None else _dev(w),
                                            store_transposed=key, renumber=renumber,
                                            vertices_array=None if vertices is None else _dev(vertices),
                                            symmetrize=not self.directed, drop_multi_edges=not self.directed)
        return self._handle, self._graphs[key]

    def number_of_vertices(self):
        src, dst, _, _, vertices = self._edges
        return int(np.unique(np.concatenate([src, dst] + ([vertices] if vertices is not None else []))).size)

    def number_of_edges(self):
        return int(self._edges[0].size)


def _frame(**cols):
    import pandas as pd
    return pd.DataFrame(cols)


def _pairs(df, value_dtype):
    """(vertices, values) device arrays of a two-column data frame 'vertex' / 'values' (pagerank.py:19-66)"""
    if df is None:
        return None, None
    return _dev(df["vertex"]), _dev(df["values"], dtype=value_dtype)


def pagerank(G: Graph, alpha=0.85, personalization=None, precomputed_vertex_out_weight=None, max_iter=100, tol=1.0e-5,
             nstart=None, dangling=None, fail_on_nonconvergence=True):
    """cugraph.pagerank (link_analysis/pagerank.py:69-330): data frame 'vertex', 'pagerank'; with fail_on_nonconvergence=False a
    tuple (data frame, converged)."""
    plc = _plc()
    h, g = G._plc_graph(True)
    vdt = np.float64 if (G.weighted and G._edges[2].dtype == np.float64) else np.float32
    pre_v, pre_w = (None, None)
    if precomputed_vertex_out_weight is not None:
        pre_v, pre_w = _dev(precomputed_vertex_out_weight["vertex"]), _dev(precomputed_vertex_out_weight["sums"], dtype=vdt)
    ns_v, ns_x = _pairs(nstart, vdt)
    if personalization is not None:
        p_v, p_x = _pairs(personalization, vdt)
        out = plc.personalized_pagerank(h, g, pre_v, pre_w, ns_v, ns_x, p_v, p_x, alpha, tol, max_iter, False,
                                        fail_on_nonconvergence=fail_on_nonconvergence)
    else:
        out = plc.pagerank(h, g, pre_v, pre_w, ns_v, ns_x, alpha, tol, max_iter, False, fail_on_nonconvergence=fail_on_nonconvergence)
    df = _frame(vertex=_host(out[0]), pagerank=_host(out[1]))
    return df if fail_on_nonconvergence else (df, bool(out[2]))


def bfs(G: Graph, start=None, depth_limit=None, i_start=None, directed=None, return_predecessors=True):
    """cugraph.bfs (traversal/bfs.py:69-330): 'vertex', 'distance'[, 'predecessor']; `start` a vertex or a list of vertices"""
    plc = _plc()
    h, g = G._plc_graph(False)
    if start is None:
        start = i_start
    starts = np.atleast_1d(np.asarray(start, dtype=G._edges[0].dtype))
    dist, pred, verts = plc.bfs(h, g, _dev(starts), not G.directed, -1 if depth_limit is None else int(depth_limit),
                                bool(return_predecessors), False)
    cols = dict(vertex=_host(verts), distance=_host(dist))
    if return_predecessors:
        cols["predecessor"] = _host(pred)
    return _frame(**cols)


def multi_source_bfs(G: Graph, sources, components=None, depth_limit=None, offload=False):
    """cugraph.multi_source_bfs (traversal/ms_bfs.py): a BFS from each source; data frame 'vertex', then 'distance_<s>' and
    'predecessor_<s>' for each source s in the order given.  The edge-list forms the reference documents for `components`
    and `offload=True` are not built.  At least one source, no duplicates, no more sources than vertices."""
    from cugraph_b200.traversal import multi_source_bfs as ms_bfs
    if components is not None:
        raise NotImplementedError("multi_source_bfs with components (BFS edge lists per source) is not implemented")
    if offload:
        raise NotImplementedError("multi_source_bfs with offload=True (results written to disk) is not implemented")
    starts = np.atleast_1d(np.asarray(sources, dtype=G._edges[0].dtype))
    if starts.size == 0:
        raise ValueError("multi_source_bfs needs at least one source")
    if np.unique(starts).size != starts.size:
        raise ValueError("multi_source_bfs sources must be distinct: each names a column pair")
    if starts.size > G.number_of_vertices():
        raise ValueError("multi_source_bfs takes at most as many sources as the graph has vertices")
    h, g = G._plc_graph(False)
    dist, pred, verts = ms_bfs(h, g, _dev(starts), -1 if depth_limit is None else int(depth_limit), True)
    dist, pred = _host(dist), _host(pred)
    cols = dict(vertex=_host(verts))
    for k, s in enumerate(starts.tolist()):
        cols[f"distance_{s}"] = dist[k]
        cols[f"predecessor_{s}"] = pred[k]
    return _frame(**cols)


def sssp(G: Graph, source=None, method=None, directed=None, return_predecessors=None, unweighted=None, overwrite=None,
         indices=None, cutoff=None):
    """cugraph.sssp (traversal/sssp.py:108-330): 'vertex', 'distance', 'predecessor'; the graph must be weighted"""
    plc = _plc()
    if not G.weighted:
        raise RuntimeError("'SSSP' requires the input graph to be weighted. 'BFS' should be used instead of 'SSSP' for unweighted graphs.")
    h, g = G._plc_graph(False)
    cut = float(np.finfo(np.float64).max) if cutoff is None else float(cutoff)
    verts, dist, pred = plc.sssp(h, g, source, cut, True, False)
    return _frame(vertex=_host(verts), distance=_host(dist), predecessor=_host(pred))


def katz_centrality(G: Graph, alpha=None, beta=1.0, max_iter=100, tol=1.0e-6, nstart=None, normalized=True):
    """cugraph.katz_centrality (centrality/katz_centrality.py): 'vertex', 'katz_centrality'.  alpha defaults to
    1 / (1 + the largest degree), as the reference documents."""
    plc = _plc()
    h, g = G._plc_graph(True)
    if alpha is None:
        src, dst, _, _, _ = G._edges
        ends = np.concatenate([src, dst]) if not G.directed else dst
        alpha = 1.0 / (1.0 + float(np.unique(ends, return_counts=True)[1].max()))
    verts, vals = plc.katz_centrality(h, g, None, alpha, beta, tol, max_iter, False)
    return _frame(vertex=_host(verts), katz_centrality=_host(vals))


def eigenvector_centrality(G: Graph, max_iter=100, tol=1.0e-6):
    """cugraph.eigenvector_centrality (centrality/eigenvector_centrality.py): 'vertex', 'eigenvector_centrality'"""
    plc = _plc()
    h, g = G._plc_graph(True)
    verts, vals = plc.eigenvector_centrality(h, g, tol, max_iter, False)
    return _frame(vertex=_host(verts), eigenvector_centrality=_host(vals))


def hits(G: Graph, max_iter=100, tol=1.0e-5, nstart=None, normalized=True):
    """cugraph.hits (link_analysis/hits.py): 'vertex', 'hubs', 'authorities'"""
    plc = _plc()
    h, g = G._plc_graph(True)
    vdt = np.float64 if (G.weighted and G._edges[2].dtype == np.float64) else np.float32
    ns_v = ns_x = None
    if nstart is not None:
        ns_v, ns_x = _dev(nstart["vertex"]), _dev(nstart["values"], dtype=vdt)
    verts, hubs, auth = plc.hits(h, g, tol, max_iter, ns_v, ns_x, normalized, False)
    return _frame(vertex=_host(verts), hubs=_host(hubs), authorities=_host(auth))


def _bc_k(G: Graph, k):
    """k as the pylibcugraph layer takes it: None, an int, or the listed vertices on the device"""
    if k is None or isinstance(k, (int, np.integer)):
        return None if k is None else int(k)
    return _dev(np.atleast_1d(np.asarray(k, dtype=G._edges[0].dtype)))


def betweenness_centrality(G: Graph, k=None, normalized=True, weight=None, endpoints=False, seed=None, random_state=None,
                           result_dtype=np.float64):
    """cugraph.betweenness_centrality (centrality/betweenness_centrality.py): 'vertex', 'betweenness_centrality'.  k: None
    (every vertex a source), an int (that many sources drawn with random_state) or a list of vertices.  Edge weights are
    not used; `weight` raises NotImplementedError, as in the reference."""
    if weight is not None:
        raise NotImplementedError("weighted implementation of betweenness centrality not currently supported")
    if result_dtype not in (np.float32, np.float64):
        raise TypeError("result type can only be np.float32 or np.float64")
    plc = _plc()
    h, g = G._plc_graph(False)
    verts, vals = plc.betweenness_centrality(h, g, _bc_k(G, k), random_state, normalized, endpoints, False)
    return _frame(vertex=_host(verts), betweenness_centrality=_host(vals).astype(result_dtype))


def edge_betweenness_centrality(G: Graph, k=None, normalized=True, weight=None, seed=None, result_dtype=np.float64):
    """cugraph.edge_betweenness_centrality: 'src', 'dst', 'betweenness_centrality'.  On an undirected graph the two
    directions of an edge are folded into one row (src < dst) holding their sum, as the reference does."""
    if weight is not None:
        raise NotImplementedError("weighted implementation of edge betweenness centrality not currently supported")
    if result_dtype not in (np.float32, np.float64):
        raise TypeError("result type can only be np.float32 or np.float64")
    plc = _plc()
    h, g = G._plc_graph(False)
    src, dst, vals, _ = plc.edge_betweenness_centrality(h, g, _bc_k(G, k), seed, normalized, False)
    df = _frame(src=_host(src), dst=_host(dst), betweenness_centrality=_host(vals).astype(result_dtype))
    if not G.directed:
        lower = df["src"] >= df["dst"]
        df.loc[lower, ["src", "dst"]] = df.loc[lower, ["dst", "src"]].to_numpy()
        df = df.groupby(by=["src", "dst"]).sum().reset_index()
    return df


def weakly_connected_components(G: Graph, directed=None, connection=None, return_labels=None):
    """cugraph.weakly_connected_components (components/connectivity.py): 'vertex', 'labels'.  The graph must be undirected."""
    plc = _plc()
    h, g = G._plc_graph(False)
    verts, labels = plc.weakly_connected_components(h, g, None, None, None, None, False)
    return _frame(vertex=_host(verts), labels=_host(labels))


def strongly_connected_components(G: Graph, directed=None, connection=None, return_labels=None):
    """cugraph.strongly_connected_components (components/connectivity.py): 'vertex', 'labels'.  The graph must be directed:
    an undirected Graph is symmetric, and the library rejects symmetric graphs here as the reference does."""
    plc = _plc()
    h, g = G._plc_graph(False)
    verts, labels = plc.strongly_connected_components(h, g, None, None, None, None, False)
    return _frame(vertex=_host(verts), labels=_host(labels))
