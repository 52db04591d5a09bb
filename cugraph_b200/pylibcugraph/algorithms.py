"""pagerank / personalized_pagerank / bfs / sssp with the reference's Python signatures
(python/pylibcugraph/pylibcugraph/{pagerank.pyx:49-59, personalized_pagerank.pyx:49-61,
bfs.pyx:50-52, sssp.pyx:48-53})."""
import ctypes as C

from cugraph_b200 import _capi
from cugraph_b200.pylibcugraph.exceptions import FailedToConvergeError
from cugraph_b200.pylibcugraph.utils import View, assert_CAI_type, copy_to_torch

INT32_MAX = 2**31 - 1


def _centrality_result(handle, res):
    L = _capi.lib()
    verts = copy_to_torch(handle, L.cugraph_centrality_result_get_vertices(res))
    vals = copy_to_torch(handle, L.cugraph_centrality_result_get_values(res))
    conv = bool(L.cugraph_centrality_result_converged(res))
    iters = int(L.cugraph_centrality_result_get_num_iterations(res))
    L.cugraph_centrality_result_free(res)
    return verts, vals, conv, iters


def pagerank(resource_handle, graph, precomputed_vertex_out_weight_vertices, precomputed_vertex_out_weight_sums,
             initial_guess_vertices, initial_guess_values, alpha, epsilon, max_iterations, do_expensive_check,
             fail_on_nonconvergence=True):
    """Returns (vertices, pageranks), or (vertices, pageranks, converged) when
    fail_on_nonconvergence is False — pagerank.pyx:150-245."""
    for a, nm in ((precomputed_vertex_out_weight_vertices, "precomputed_vertex_out_weight_vertices"),
                  (precomputed_vertex_out_weight_sums, "precomputed_vertex_out_weight_sums"),
                  (initial_guess_vertices, "initial_guess_vertices"), (initial_guess_values, "initial_guess_values")):
        assert_CAI_type(a, nm, True)
    views = [View(a) for a in (precomputed_vertex_out_weight_vertices, precomputed_vertex_out_weight_sums,
                               initial_guess_vertices, initial_guess_values)]
    res = C.c_void_p()
    err = C.c_void_p()
    resource_handle.order_after_caller()
    code = _capi.lib().cugraph_pagerank_allow_nonconvergence(
        resource_handle.ptr, graph.ptr, views[0].ptr, views[1].ptr, views[2].ptr, views[3].ptr,
        float(alpha), float(epsilon), int(max_iterations), int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    for v in views:
        v.free()
    _capi.check(code, err, "cugraph_pagerank_allow_nonconvergence")
    verts, vals, conv, _ = _centrality_result(resource_handle, res)
    if fail_on_nonconvergence:
        if not conv:
            raise FailedToConvergeError
        return (verts, vals)
    return (verts, vals, conv)


def personalized_pagerank(resource_handle, graph, precomputed_vertex_out_weight_vertices,
                          precomputed_vertex_out_weight_sums, initial_guess_vertices, initial_guess_values,
                          personalization_vertices, personalization_values, alpha, epsilon, max_iterations,
                          do_expensive_check, fail_on_nonconvergence=True):
    assert_CAI_type(personalization_vertices, "personalization_vertices", True)
    assert_CAI_type(personalization_values, "personalization_values", True)
    views = [View(a) for a in (precomputed_vertex_out_weight_vertices, precomputed_vertex_out_weight_sums,
                               initial_guess_vertices, initial_guess_values, personalization_vertices,
                               personalization_values)]
    res = C.c_void_p()
    err = C.c_void_p()
    resource_handle.order_after_caller()
    code = _capi.lib().cugraph_personalized_pagerank_allow_nonconvergence(
        resource_handle.ptr, graph.ptr, *[v.ptr for v in views], float(alpha), float(epsilon),
        int(max_iterations), int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    for v in views:
        v.free()
    _capi.check(code, err, "cugraph_personalized_pagerank_allow_nonconvergence")
    verts, vals, conv, _ = _centrality_result(resource_handle, res)
    if fail_on_nonconvergence:
        if not conv:
            raise FailedToConvergeError
        return (verts, vals)
    return (verts, vals, conv)


def _paths_result(handle, res, want_pred=True):
    L = _capi.lib()
    verts = copy_to_torch(handle, L.cugraph_paths_result_get_vertices(res))
    dist = copy_to_torch(handle, L.cugraph_paths_result_get_distances(res))
    pred = copy_to_torch(handle, L.cugraph_paths_result_get_predecessors(res))
    L.cugraph_paths_result_free(res)
    return verts, dist, pred


def bfs(handle, graph, sources, direction_optimizing, depth_limit, compute_predecessors, do_expensive_check):
    """Returns (distances, predecessors, vertices) — bfs.pyx:140-200 (note the order)."""
    assert_CAI_type(sources, "sources")
    if depth_limit <= 0:
        depth_limit = INT32_MAX - 1  # bfs.pyx:144-145
    sv = View(sources)
    res = C.c_void_p()
    err = C.c_void_p()
    handle.order_after_caller()
    code = _capi.lib().cugraph_bfs(handle.ptr, graph.ptr, sv.ptr, int(bool(direction_optimizing)), int(depth_limit),
                                   int(bool(compute_predecessors)), int(bool(do_expensive_check)),
                                   C.byref(res), C.byref(err))
    sv.free()
    _capi.check(code, err, "cugraph_bfs")
    verts, dist, pred = _paths_result(handle, res)
    return (dist, pred, verts)


def sssp(resource_handle, graph, source, cutoff, compute_predecessors, do_expensive_check):
    """Returns (vertices, distances, predecessors) — sssp.pyx:120-170."""
    res = C.c_void_p()
    err = C.c_void_p()
    resource_handle.order_after_caller()
    code = _capi.lib().cugraph_sssp(resource_handle.ptr, graph.ptr, int(source), float(cutoff),
                                    int(bool(compute_predecessors)), int(bool(do_expensive_check)),
                                    C.byref(res), C.byref(err))
    _capi.check(code, err, "cugraph_sssp")
    verts, dist, pred = _paths_result(resource_handle, res)
    return (verts, dist, pred)


def katz_centrality(resource_handle, graph, betas, alpha, beta, epsilon, max_iterations, do_expensive_check):
    """Returns (vertices, values) — katz_centrality.pyx:47-145.  `betas` is accepted and, as in the reference's C entry
    point (c_api/katz.cpp:151-152), not used: every vertex gets `beta`."""
    assert_CAI_type(betas, "betas", allow_none=True)
    bv = View(betas)
    res, err = C.c_void_p(), C.c_void_p()
    resource_handle.order_after_caller()
    code = _capi.lib().cugraph_katz_centrality(resource_handle.ptr, graph.ptr, bv.ptr, float(alpha), float(beta), float(epsilon),
                                               int(max_iterations), int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    bv.free()
    _capi.check(code, err, "cugraph_katz_centrality")
    verts, vals, _, _ = _centrality_result(resource_handle, res)
    return (verts, vals)


def eigenvector_centrality(resource_handle, graph, epsilon, max_iterations, do_expensive_check):
    """Returns (vertices, values) — eigenvector_centrality.pyx."""
    res, err = C.c_void_p(), C.c_void_p()
    resource_handle.order_after_caller()
    code = _capi.lib().cugraph_eigenvector_centrality(resource_handle.ptr, graph.ptr, float(epsilon), int(max_iterations),
                                                      int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    _capi.check(code, err, "cugraph_eigenvector_centrality")
    verts, vals, _, _ = _centrality_result(resource_handle, res)
    return (verts, vals)


def hits(resource_handle, graph, tol, max_iter, initial_hubs_guess_vertices, initial_hubs_guess_values, normalized,
         do_expensive_check):
    """Returns (vertices, hubs, authorities) — hits.pyx:49-184."""
    assert_CAI_type(initial_hubs_guess_vertices, "initial_hubs_guess_vertices", allow_none=True)
    assert_CAI_type(initial_hubs_guess_values, "initial_hubs_guess_values", allow_none=True)
    gv, gx = View(initial_hubs_guess_vertices), View(initial_hubs_guess_values)
    res, err = C.c_void_p(), C.c_void_p()
    resource_handle.order_after_caller()
    L = _capi.lib()
    code = L.cugraph_hits(resource_handle.ptr, graph.ptr, float(tol), int(max_iter), gv.ptr, gx.ptr, int(bool(normalized)),
                          int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    gv.free()
    gx.free()
    _capi.check(code, err, "cugraph_hits")
    verts = copy_to_torch(resource_handle, L.cugraph_hits_result_get_vertices(res))
    hubs = copy_to_torch(resource_handle, L.cugraph_hits_result_get_hubs(res))
    auth = copy_to_torch(resource_handle, L.cugraph_hits_result_get_authorities(res))
    L.cugraph_hits_result_free(res)
    return (verts, hubs, auth)


def _ensure_wcc_args(graph, offsets, indices, weights, labels):
    """argument rules of weakly_connected_components.pyx:49-104"""
    if graph is not None:
        bad = [p for p in (offsets, indices, weights) if p is not None]
        kind = "graph"
    else:
        bad = [p for p in (offsets, indices) if p is None]
        kind = "csr_arrays"
    if bad:
        raise TypeError("Invalid input combination: Must set either 'graph' or "
                        "a combination of 'offsets', 'indices' and 'weights', not both")
    if kind == "csr_arrays":
        assert_CAI_type(offsets, "offsets")
        assert_CAI_type(indices, "indices")
        assert_CAI_type(weights, "weights", True)
    if labels is not None:
        assert_CAI_type(labels, "labels")
        if kind == "csr_arrays":
            import numpy as np
            odt, idt, ldt = (np.dtype(a.__cuda_array_interface__["typestr"]) for a in (offsets, indices, labels))
            if odt != idt:
                raise TypeError(f"offsets dtype must match indices dtype (got offsets.dtype={odt!r}, indices.dtype={idt!r})")
            if ldt != idt:
                raise TypeError(f"labels dtype must match indices dtype (got labels.dtype={ldt!r}, indices.dtype={idt!r})")
    return kind


def _labeling(fn_name, resource_handle, graph, offsets, indices, weights, labels, do_expensive_check, is_symmetric):
    """the legacy CSR form (a graph built from offsets / indices [/ weights] with renumber=False), the C call and the result
    plumbing shared by weakly_connected_components and strongly_connected_components"""
    from cugraph_b200.pylibcugraph.graph_properties import GraphProperties
    from cugraph_b200.pylibcugraph.graphs import SGGraph
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    kind = _ensure_wcc_args(graph, offsets, indices, weights, labels)
    if kind == "csr_arrays":
        if resource_handle is None:
            resource_handle = ResourceHandle()
        graph = SGGraph(resource_handle, GraphProperties(is_symmetric=is_symmetric, is_multigraph=False), offsets, indices,
                        weights, store_transposed=False, renumber=False, do_expensive_check=True, input_array_format="CSR")
    res, err = C.c_void_p(), C.c_void_p()
    resource_handle.order_after_caller()
    L = _capi.lib()
    code = getattr(L, fn_name)(resource_handle.ptr, graph.ptr, int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    _capi.check(code, err, fn_name)
    verts = copy_to_torch(resource_handle, L.cugraph_labeling_result_get_vertices(res))
    labs = copy_to_torch(resource_handle, L.cugraph_labeling_result_get_labels(res))
    L.cugraph_labeling_result_free(res)
    if labels is not None:
        import torch
        out = torch.as_tensor(labels, device=labs.device) if not isinstance(labels, torch.Tensor) else labels
        out.copy_(labs)   # renumber=False: the result rows are in vertex order
        return None
    return (verts, labs)


def weakly_connected_components(resource_handle, graph, offsets, indices, weights, labels, do_expensive_check):
    """weakly_connected_components.pyx:107-290.  Either `graph`, or the CSR arrays `offsets` / `indices` [/ `weights`] of a
    symmetric graph (the legacy form: a graph is built from them with renumber=False).  Returns (vertices, labels); with a
    `labels` array the labels are written into it (vertex order) and None is returned."""
    return _labeling("cugraph_weakly_connected_components", resource_handle, graph, offsets, indices, weights, labels,
                     do_expensive_check, is_symmetric=True)


def strongly_connected_components(resource_handle, graph, offsets, indices, weights, labels, do_expensive_check):
    """strongly_connected_components.pyx:107-270.  Either `graph` (not symmetric), or the CSR arrays `offsets` / `indices`
    [/ `weights`] of a directed graph (the legacy form: a graph is built from them with is_symmetric=False,
    is_multigraph=False, store_transposed=False, renumber=False).  Returns (vertices, labels); with a `labels` array the
    labels are written into it (vertex order) and None is returned.  Weights are ignored."""
    return _labeling("cugraph_strongly_connected_components", resource_handle, graph, offsets, indices, weights, labels,
                     do_expensive_check, is_symmetric=False)


def generate_rmat_edgelist(resource_handle, random_state, scale, num_edges, a, b, c, clip_and_flip, scramble_vertex_ids,
                           include_edge_weights, minimum_weight, maximum_weight, dtype, include_edge_ids, include_edge_types,
                           min_edge_type_value, max_edge_type_value, multi_gpu):
    """generate_rmat_edgelist.pyx: returns (sources, destinations, weights | None, edge ids | None, edge types | None).
    The edges come from the library's device generator (the reference's sampling rule over a counter-based stream seeded with
    `random_state`), weights / types from its uniform generator; ids are 0 .. num_edges-1 (as the reference numbers them).
    multi_gpu=True (on the default torch.distributed group): num_edges is this rank's count, and the rank generates edges
    [start, start + num_edges) of the same stream, start = the sum of the counts of the lower ranks (one all-gather, as the
    reference numbers multi-GPU edge ids); weights and types are drawn at the same global indices and ids are start + k.
    The ranks' outputs in rank order are then one single-GPU call over the total count, bit for bit."""
    import numpy as np
    import torch
    L = _capi.lib()
    dev = "cuda" if torch.cuda.is_available() else "cpu"
    seed = int(random_state) if random_state is not None else 0
    start, total = 0, int(num_edges)
    if multi_gpu:
        from cugraph_b200 import mg
        mine = torch.tensor([int(num_edges)], dtype=torch.int64, device=dev)
        counts = torch.empty(mg.dist.get_world_size(), dtype=torch.int64, device=dev)
        mg.all_gather_into(counts, mine, None)
        counts = counts.tolist()
        start, total = sum(counts[:mg.dist.get_rank()]), sum(counts)
    src = torch.empty(num_edges, dtype=torch.int32, device=dev)
    dst = torch.empty(num_edges, dtype=torch.int32, device=dev)
    vs, vd, err = View(src), View(dst), C.c_void_p()
    resource_handle.order_after_caller()
    code = L.cugraph_b200_generate_rmat_edgelist_at(resource_handle.ptr, int(scale), start, int(num_edges), float(a), float(b),
                                                    float(c), seed, int(bool(clip_and_flip)), int(bool(scramble_vertex_ids)),
                                                    vs.ptr, vd.ptr, C.byref(err))
    vs.free()
    vd.free()
    _capi.check(code, err, "cugraph_b200_generate_rmat_edgelist_at")

    def uniform(tdtype, lo, hi, salt):
        out = torch.empty(num_edges, dtype=tdtype, device=dev)
        vo, e2 = View(out), C.c_void_p()
        c2 = L.cugraph_b200_generate_uniform_at(resource_handle.ptr, seed + salt, start, float(lo), float(hi), vo.ptr,
                                                C.byref(e2))
        vo.free()
        _capi.check(c2, e2, "cugraph_b200_generate_uniform_at")
        return out

    weights = ids = types = None
    if include_edge_weights:
        tdt = torch.float64 if np.dtype(dtype) == np.float64 else torch.float32
        weights = uniform(tdt, minimum_weight, maximum_weight, 0x9E37)
    if include_edge_ids:
        ids = torch.arange(start, start + int(num_edges), dtype=torch.int64 if multi_gpu and total > 2**31 else torch.int32,
                           device=dev)
    if include_edge_types:
        types = uniform(torch.int32, min_edge_type_value, max_edge_type_value + 1, 0x79B9)
    import torch as _t
    if _t.cuda.is_available():
        _t.cuda.synchronize()
    return (src, dst, weights, ids, types)


def _degrees(fn_name, resource_handle, graph, source_vertices, do_expensive_check):
    assert_CAI_type(source_vertices, "source_vertices", allow_none=True)
    sv = View(source_vertices)
    res, err = C.c_void_p(), C.c_void_p()
    resource_handle.order_after_caller()
    L = _capi.lib()
    code = getattr(L, fn_name)(resource_handle.ptr, graph.ptr, sv.ptr, int(bool(do_expensive_check)), C.byref(res), C.byref(err))
    sv.free()
    _capi.check(code, err, fn_name)
    verts = copy_to_torch(resource_handle, L.cugraph_degrees_result_get_vertices(res))
    vin, vout = L.cugraph_degrees_result_get_in_degrees(res), L.cugraph_degrees_result_get_out_degrees(res)
    ins = copy_to_torch(resource_handle, vin) if vin else None
    outs = copy_to_torch(resource_handle, vout) if vout else None
    L.cugraph_degrees_result_free(res)
    return verts, ins, outs


def in_degrees(resource_handle, graph, source_vertices, do_expensive_check):
    """Returns (vertices, in degrees) — degrees.pyx"""
    v, i, _ = _degrees("cugraph_in_degrees", resource_handle, graph, source_vertices, do_expensive_check)
    return (v, i)


def out_degrees(resource_handle, graph, source_vertices, do_expensive_check):
    """Returns (vertices, out degrees) — degrees.pyx"""
    v, _, o = _degrees("cugraph_out_degrees", resource_handle, graph, source_vertices, do_expensive_check)
    return (v, o)


def degrees(resource_handle, graph, source_vertices, do_expensive_check):
    """Returns (vertices, in degrees, out degrees) — degrees.pyx"""
    return _degrees("cugraph_degrees", resource_handle, graph, source_vertices, do_expensive_check)
