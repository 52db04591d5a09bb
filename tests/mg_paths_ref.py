"""Multi-GPU BFS from a set of sources and MGGraph.extract_paths on every rank of a grid in ONE process (tests/mg_world.py:
the drivers themselves), the single-GPU references, a numpy restatement of single GPU's k_paths_max_len / k_paths_walk
(traverse.cu), the graphs and the checks.

Shared by tests/test_mg_paths_cpu.py and tests/test_mg_paths_gpu.py."""
import ctypes as C

import numpy as np

import oracle
from tests import mg_world

IMAX = np.iinfo(np.int32).max


def _errors(fn, *args):
    """fn(*args), or the (type name, message) of what it raised"""
    try:
        return fn(*args)
    except Exception as e:  # noqa: BLE001
        return type(e).__name__, str(e)


def _worker(rank, world, s, d, sources, dests, depth_limit, device, repeat):
    import torch
    g = mg_world.graph(rank, world, s, d, device=device)
    src = sources[rank] if isinstance(sources, list) else sources
    if isinstance(src, np.ndarray):
        src = torch.as_tensor(src).to(device)
    v, dist, pred = g.bfs(src, depth_limit)
    out = dict(v=v.cpu().numpy(), dist=dist.cpu().numpy(), pred=pred.cpu().numpy(), n_local=g.part.n_local)
    if dests is not None:
        dst = torch.as_tensor(dests[rank]).to(device)
        paths, length = g.extract_paths(dist, pred, dst)
        out.update(paths=paths.cpu().numpy(), length=length, rounds=g.last_paths_stats["rounds"])
        if repeat:
            again, length2 = g.extract_paths(dist, pred, dst)
            out.update(again=again.cpu().numpy(), length2=length2)
    return out


def mg_bfs_paths(s, d, world, sources, dests=None, depth_limit=-1, device="cpu", repeat=False):
    """MGGraph.bfs(sources) on `world` ranks (sources: one id for every rank, or a list of per-rank id arrays), then, with
    `dests` (a list of per-rank id arrays), MGGraph.extract_paths of each rank's destinations (twice with `repeat`).
    Returns the ranks' dicts (v, dist, pred, n_local[, paths, length, rounds[, again, length2]])."""
    return mg_world.run(world, _worker, s, d, sources, dests, depth_limit, device, repeat)


def gather(res):
    """(vertex ids, distances, predecessors) of every rank, concatenated"""
    return (np.concatenate([r["v"] for r in res]).astype(np.int64), np.concatenate([r["dist"] for r in res]),
            np.concatenate([r["pred"] for r in res]).astype(np.int64))


def check_bfs(s, d, res, sources, depth_limit=-1):
    """distances bit-exact against the oracle from the union of `sources` on the graph's vertices (the ids of the edges),
    predecessors by the reference's predicate (bfs_test.cpp:213-233)"""
    vids, dist, pred = gather(res)
    ids, remap = mg_world.present(s, d, int(max(s.max(), d.max())) + 1)
    assert np.array_equal(np.sort(vids), ids)
    srcs = remap[np.unique(np.asarray(sources, np.int64))].astype(np.int32)
    ref_d, _ = oracle.bfs(remap[s].astype(np.int32), remap[d].astype(np.int32), ids.size, srcs,
                          depth_limit=None if depth_limit < 0 else depth_limit)
    ref_d = np.asarray(ref_d, np.int64)
    ref_d = np.where((ref_d < 0) | (ref_d >= IMAX), IMAX, ref_d)
    got_d = np.full(ids.size, -5, np.int64)
    got_p = np.full(ids.size, -5, np.int64)
    got_d[remap[vids]] = dist
    got_p[remap[vids]] = np.where(pred >= 0, remap[np.maximum(pred, 0)], -1)
    assert np.array_equal(got_d, ref_d)
    assert oracle.check_bfs_predecessors(remap[s], remap[d], ids.size, got_d.astype(np.int32), got_p, srcs)
    return got_d


def paths_reference(vids, dist, pred, dests):
    """single GPU's k_paths_max_len / k_paths_walk restated over external ids: (paths [len(dests), length], length).  vids,
    dist and pred are a BFS result (predecessors as external ids); dests any external ids"""
    vids = np.asarray(vids, np.int64)
    order = np.argsort(vids)
    sv = vids[order]

    def internal(x):   # ext_to_int: -1 for an id that is not a vertex
        x = np.asarray(x, np.int64)
        if sv.size == 0:
            return np.full(x.shape, -1, np.int64)
        pos = np.searchsorted(sv, x).clip(max=sv.size - 1)
        return np.where(sv[pos] == x, order[pos], -1)

    pred_i = internal(pred)
    dest_i = internal(dests)
    dist = np.asarray(dist, np.int64)
    top = 0
    for v in dest_i.tolist():
        if v < 0 or pred_i[v] < 0 or dist[v] >= IMAX:
            continue
        top = max(top, int(dist[v]))
    length = top + 1
    paths = np.full((dest_i.size, length), -1, np.int64)
    for i, v in enumerate(dest_i.tolist()):
        if v < 0:
            continue
        k = int(dist[v])
        if k >= IMAX or k >= length:
            continue
        while k >= 0 and v >= 0:
            paths[i, k] = vids[v]
            v = int(pred_i[v])
            k -= 1
    return paths, length


def check_paths(res, dests):
    """every rank's rows = the restatement applied to the gathered BFS result and the concatenated destinations, the same
    max_path_length on every rank, `length - 1` rounds; with `again`: a second call gave the same.  Returns (paths of all
    ranks concatenated, length)."""
    vids, dist, pred = gather(res)
    want, length = paths_reference(vids, dist, pred, np.concatenate([np.asarray(x, np.int64) for x in dests]))
    at = 0
    for r, x in zip(res, dests):
        assert r["length"] == length
        assert r["rounds"] == length - 1
        assert r["paths"].shape == (len(x), length)
        assert r["paths"].dtype == r["v"].dtype
        assert np.array_equal(r["paths"], want[at:at + len(x)])
        if "again" in r:
            assert r["length2"] == length and np.array_equal(r["again"], r["paths"])
        at += len(x)
    return want, length


def split(ids, world, rng):
    """ids dealt to `world` ranks in random sizes (some possibly empty), as int32 arrays"""
    cuts = np.sort(rng.integers(0, len(ids) + 1, world - 1))
    return [np.asarray(x, np.int32) for x in np.split(np.asarray(ids), cuts)]


def owned_by(ids, world):
    """the rank that owns every id (mg.vertex_owner)"""
    import torch
    from cugraph_b200 import mg
    return mg.vertex_owner(torch.as_tensor(np.asarray(ids, np.int64)), world).numpy()


# ---------------------------------------------------------------------------------------------------- single GPU
def single_gpu_paths(s, d, sources, dests, vertex_dtype=np.int32):
    """cugraph_bfs from `sources` and cugraph_extract_paths of `dests` on the single-GPU graph of the same edges (its
    vertices: the ids of the edges): (distances by vertex, paths [len(dests), length])"""
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View, copy_to_torch
    from tests.gpu_util import make_graph
    h, g = make_graph(s, d, vertex_dtype=vertex_dtype)
    L = _capi.lib()
    sv = View(torch.as_tensor(np.asarray(sources, vertex_dtype)).cuda())
    dv = View(torch.as_tensor(np.asarray(dests, vertex_dtype)).cuda())
    res, out, err = C.c_void_p(), C.c_void_p(), C.c_void_p()
    h.order_after_caller()
    _capi.check(L.cugraph_bfs(h.ptr, g.ptr, sv.ptr, 0, IMAX - 1, 1, 0, C.byref(res), C.byref(err)), err, "cugraph_bfs")
    verts = copy_to_torch(h, L.cugraph_paths_result_get_vertices(res)).cpu().numpy()
    dist = copy_to_torch(h, L.cugraph_paths_result_get_distances(res)).cpu().numpy()
    code = L.cugraph_extract_paths(h.ptr, g.ptr, sv.ptr, res, dv.ptr, C.byref(out), C.byref(err))
    L.cugraph_paths_result_free(res)
    _capi.check(code, err, "cugraph_extract_paths")
    n = int(L.cugraph_extract_paths_result_get_max_path_length(out))
    paths = copy_to_torch(h, L.cugraph_extract_paths_result_get_paths(out)).cpu().numpy().reshape(len(dests), n)
    L.cugraph_extract_paths_result_free(out)
    sv.free()
    dv.free()
    by_id = np.full(int(verts.max()) + 1 if verts.size else 0, -5, np.int64)
    by_id[verts] = dist
    return by_id, paths


# ---------------------------------------------------------------------------------------------------- graphs
def rmat_graph(scale, seed=700):
    """directed RMAT, ef 16: unreached parts for most sources"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed + scale)
    return np.asarray(s, np.int32), np.asarray(d, np.int32)


def forced_graph(n_tree=600, n_roots=5, n_cycle=40, seed=3):
    """a directed forest whose every reached vertex has exactly ONE in-neighbour one level closer to the roots, so that
    BFS predecessors are forced: out-trees from n_roots roots (every other tree vertex hangs below a random earlier one),
    edges from vertices back to their tree's root, and a directed cycle that no root reaches, with edges into the trees.
    Ids are scattered.  Returns (s, d, roots, unreached ids)."""
    rng = np.random.default_rng(seed)
    parent = np.full(n_tree, -1)
    root_of = np.arange(n_tree)
    for v in range(n_roots, n_tree):
        parent[v] = rng.integers(0, v)
        root_of[v] = root_of[parent[v]]
    kids = np.arange(n_roots, n_tree)
    back = rng.choice(kids, n_tree // 5, replace=False)
    cyc = n_tree + np.arange(n_cycle)
    into = rng.choice(n_tree, n_cycle // 2, replace=False)
    s = np.concatenate([parent[kids], back, cyc, cyc[:n_cycle // 2]])
    d = np.concatenate([kids, root_of[back], np.roll(cyc, -1), into])
    perm = rng.permutation(n_tree + n_cycle + 7) + 3          # ids 0..2 and a few others are not vertices
    return perm[s].astype(np.int32), perm[d].astype(np.int32), perm[:n_roots].astype(np.int32), perm[cyc].astype(np.int32)


def not_vertices(s, d, k=3):
    """k ids that are not vertices of the graph of these edges"""
    used = set(np.concatenate([s, d]).tolist())
    out, x = [], 0
    while len(out) < k:
        if x not in used:
            out.append(x)
        x += 1
    return np.asarray(out, np.int32)
