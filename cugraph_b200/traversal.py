"""Traversals that have no counterpart in the reference's pylibcugraph: multi-source BFS (cugraph_b200_multi_source_bfs,
csrc/traverse.cu), one BFS per source with up to 64 sources advanced by each pass over the graph."""
from __future__ import annotations

import ctypes as C

INT32_MAX = 2**31 - 1


def multi_source_bfs(handle, graph, sources, depth_limit=-1, compute_predecessors=True):
    """A BFS from each vertex of `sources` (a device array of the graph's vertex type) on a `pylibcugraph.SGGraph`.

    Returns (distances, predecessors, vertices), the order of `pylibcugraph.bfs`, as torch CUDA tensors: distances has shape
    [len(sources), V] and row s equals the distances `pylibcugraph.bfs` returns for the one source sources[s] (the vertex
    type, INT32_MAX / INT64_MAX where unreached); predecessors has the same shape (-1 for the source and unreached vertices),
    or is None without compute_predecessors; vertices (V) orders the columns.  depth_limit <= 0: no limit."""
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.algorithms import _paths_result
    from cugraph_b200.pylibcugraph.utils import View, assert_CAI_type
    assert_CAI_type(sources, "sources")
    if depth_limit <= 0:
        depth_limit = INT32_MAX - 1
    sv = View(sources)
    res = C.c_void_p()
    err = C.c_void_p()
    handle.order_after_caller()
    code = _capi.lib().cugraph_b200_multi_source_bfs(handle.ptr, graph.ptr, sv.ptr, int(depth_limit),
                                                     int(bool(compute_predecessors)), C.byref(res), C.byref(err))
    sv.free()
    _capi.check(code, err, "cugraph_b200_multi_source_bfs")
    verts, dist, pred = _paths_result(handle, res)
    dist = dist.reshape(len(sources), verts.numel())
    pred = pred.reshape(len(sources), verts.numel()) if compute_predecessors else None
    return dist, pred, verts
