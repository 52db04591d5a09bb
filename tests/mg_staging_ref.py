"""MGGraph's construction options (vertices, drop_self_loops, drop_multi_edges, symmetrize) on every rank of a grid in ONE
process (tests/mg_world.py), numpy restatements of the staging rules, the single-GPU reference, the graphs and the checks.

Shared by tests/test_mg_staging_cpu.py and tests/test_mg_staging_gpu.py."""
import ctypes as C
import itertools

import numpy as np
import torch

from tests import mg_world

OPTIONS = [dict(drop_self_loops=a, drop_multi_edges=b, symmetrize=c) for a, b, c in itertools.product((False, True), repeat=3)]
OPTION_IDS = ["".join(k[0] if v else "-" for k, v in zip("lms", o.values())) for o in OPTIONS]   # l = loops, m = multi, s = sym


# ------------------------------------------------------------------------------------------------ numpy restatements
def _pair(a, b, wt):
    """symmetrize's rule over one unordered pair: the i-th lightest of a with the i-th lightest of b -> (W)((x + y) / 2),
    the unpaired ones as they are"""
    a, b = sorted(a), sorted(b)
    out = []
    for i in range(max(len(a), len(b))):
        if i < len(a) and i < len(b):
            out.append(wt((wt(a[i]) + wt(b[i])) / wt(2)))
        else:
            out.append(a[i] if i < len(a) else b[i])
    return out


def stage_block_np(rows, cols, rev, w, drop_multi_edges, symmetrize):
    """cugraph_b200_block_stage_edges restated: the sorted list of staged (row, col, weight or 0)"""
    wt = np.float64 if w is None else w.dtype.type
    ww = np.zeros(len(rows), wt) if w is None else w
    flags = np.zeros(len(rows), np.int64) if (rev is None or not symmetrize) else (np.asarray(rev) != 0).astype(np.int64)
    groups = {}
    for r, c, f, x in zip(rows.tolist(), cols.tolist(), flags.tolist(), ww):
        groups.setdefault((r, c), ([], []))[f].append(x)
    out = []
    for (r, c), (a, b) in groups.items():
        if drop_multi_edges:
            a, b = a and [min(a)], b and [min(b)]
        ws = _pair(a, b, wt) if symmetrize else a + b
        out += [(r, c, x) for x in ws]
    return sorted(out, key=lambda e: (e[0], e[1], float(e[2])))


def stage_graph_np(s, d, w, vertices, drop_self_loops=False, drop_multi_edges=False, symmetrize=False):
    """single-GPU staging over an external-id edge list: (vertices sorted, staged (src, dst, w or None)); multi-edges keep
    their minimum"""
    s, d = np.asarray(s, np.int64), np.asarray(d, np.int64)
    wt = np.float64 if w is None else w.dtype.type
    ww = np.zeros(s.size, wt) if w is None else w
    if drop_self_loops:
        keep = s != d
        s, d, ww = s[keep], d[keep], ww[keep]
    verts = np.unique(np.concatenate([s, d, np.asarray(vertices if vertices is not None else [], np.int64)]))
    edges = {}
    for u, v, x in zip(s.tolist(), d.tolist(), ww):
        edges.setdefault((u, v), []).append(x)
    if drop_multi_edges:
        edges = {k: [min(x)] for k, x in edges.items()}
    if symmetrize:
        out = {}
        for (u, v) in edges:
            lo, hi = min(u, v), max(u, v)
            if (lo, hi) in out:
                continue
            if lo == hi:
                out[(lo, hi)] = list(edges[(lo, hi)])
                continue
            ws = _pair(edges.get((lo, hi), []), edges.get((hi, lo), []), wt)
            out[(lo, hi)] = ws
            out[(hi, lo)] = list(ws)
        edges = out
    es = [(u, v, x) for (u, v), xs in edges.items() for x in xs]
    S = np.array([e[0] for e in es], np.int64)
    D = np.array([e[1] for e in es], np.int64)
    W = None if w is None else np.array([e[2] for e in es], wt)
    return verts, (S, D, W)


def degrees_np(verts, S, D):
    """(in, out) edge counts of the staged edge list, indexed like verts"""
    pos = {int(v): i for i, v in enumerate(verts)}
    din, dout = np.zeros(verts.size, np.int64), np.zeros(verts.size, np.int64)
    for u, v in zip(S.tolist(), D.tolist()):
        dout[pos[u]] += 1
        din[pos[v]] += 1
    return din, dout


# ------------------------------------------------------------------------------------------------ the entry point
def stage_block(rows, cols, rev, w, n_rows, n_cols, drop_multi_edges, symmetrize):
    """cugraph_b200_block_stage_edges over copies of the arrays: the sorted list of staged (row, col, weight or 0)"""
    from cugraph_b200 import _capi
    from cugraph_b200.mg import _views
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    dev = "cuda"
    r = torch.as_tensor(np.asarray(rows)).to(dev).clone()
    c = torch.as_tensor(np.asarray(cols)).to(dev).clone()
    f = None if rev is None else torch.as_tensor(np.asarray(rev)).to(dev).clone()
    wt = None if w is None else torch.as_tensor(np.asarray(w)).to(dev).clone()
    handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
    n_out, err = C.c_size_t(), C.c_void_p()
    with _views(r, c, f, wt) as (rv, cv, fv, wv):
        code = _capi.lib().cugraph_b200_block_stage_edges(handle.ptr, n_rows, n_cols, rv.ptr, cv.ptr, fv.ptr, wv.ptr,
                                                          int(drop_multi_edges), int(symmetrize), C.byref(n_out), C.byref(err))
    _capi.check(code, err, "cugraph_b200_block_stage_edges")
    m = n_out.value
    R, Cc = r[:m].cpu().numpy(), c[:m].cpu().numpy()
    W = np.zeros(m) if wt is None else wt[:m].cpu().numpy()
    keys = R.astype(np.int64) * (1 << 32) + Cc
    assert (np.diff(keys) >= 0).all()                     # ordered by (row, col)
    return sorted(zip(R.tolist(), Cc.tolist(), W), key=lambda e: (e[0], e[1], float(e[2])))


def random_block(rng, n_rows, n_cols, n, wdtype):
    """block-coordinate edges with duplicates of equal and of distinct weights, reverse-flagged copies, more copies in one
    direction than the other"""
    rows = rng.integers(0, n_rows, n).astype(np.int32)
    cols = rng.integers(0, n_cols, n).astype(np.int32)
    rev = (rng.random(n) < 0.4).astype(np.uint8)
    w = None if wdtype is None else (rng.integers(1, 8, n) / 4).astype(wdtype)   # few distinct values: equal weights
    k = n // 4                                                                       # a quarter repeats earlier positions
    rows[-k:], cols[-k:] = rows[:k], cols[:k]
    if w is not None:
        w[-k:] = np.where(rng.random(k) < 0.5, w[:k], w[-k:])
    return rows, cols, rev, w


# ------------------------------------------------------------------------------------------------ MG and single GPU
def _ids(rank, world, vertex_lists):
    v = vertex_lists[rank] if vertex_lists is not None else None
    return None if v is None else torch.as_tensor(np.asarray(v))


def vertex_splits(ids, s, world):
    """ways to pass the extra vertex ids on `world` ranks: all from rank 0; all from a rank that owns none of them (None
    when every rank owns one); split over the ranks with duplicates"""
    from cugraph_b200.mg import vertex_owner
    owners = set(vertex_owner(torch.as_tensor(ids), world).tolist())
    none_owned = next((r for r in range(world) if r not in owners), None)
    out = [[ids] + [None] * (world - 1)]
    if none_owned is not None:
        out.append([ids if r == none_owned else None for r in range(world)])
    out.append([ids[r % 2::2] if r < world - 1 else np.concatenate([ids[1::2], ids[:3]]) for r in range(world)])
    return out


def _worker(rank, world, s, d, w, vertex_lists, opts, runs, device):
    from cugraph_b200 import mg
    s_, d_, *rest = mg_world.share(rank, world, s, d, *([] if w is None else [w]))
    t = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(device)  # noqa: E731
    v = _ids(rank, world, vertex_lists)
    g = mg.MGGraph(t(s_), t(d_), t(rest[0]) if rest else None, vertices=None if v is None else v.to(device), **opts)
    out = {"degrees": g.degrees()}
    for name, args in runs:
        if name == "pagerank":
            vv, x, _, _ = g.pagerank(**args)
            out[(name, str(args))] = (vv, x)
        elif name in ("bfs", "sssp"):
            vv, dd, _ = getattr(g, name)(args["source"], compute_predecessors=False)
            out[(name, str(args))] = (vv, dd)
        elif name == "wcc":
            out[(name, "")] = g.weakly_connected_components()
        elif name == "katz":
            out[(name, "")] = g.katz_centrality(**args)
        elif name == "eigenvector":
            out[(name, "")] = g.eigenvector_centrality(**args)
        elif name == "hits":
            vv, hb, au = g.hits(**args)
            out[(name, "")] = (vv, hb)
            out[("hits_auth", "")] = (vv, au)
    return out


def mg_run(s, d, w, world, opts, runs=(), vertex_lists=None, device="cpu"):
    """MGGraph(**opts) on `world` ranks (rank k passes vertex_lists[k]).  Returns {key: {vertex id: value}} over all ranks,
    key "in" / "out" for the degrees and (name, args) for every run; checks that no vertex is owned twice"""
    res = mg_world.run(world, _worker, s, d, w, vertex_lists, opts, list(runs), device)
    merged = {}
    for r in res:
        vv, din, dout = r.pop("degrees")
        assert din.dtype == vv.dtype and dout.dtype == vv.dtype
        for key, (v, x) in [("in", (vv, din)), ("out", (vv, dout))] + list(r.items()):
            m = merged.setdefault(key, {})
            for a, b in zip(v.cpu().tolist(), x.cpu().numpy()):
                assert a not in m
                m[a] = b
    return merged


def single_gpu(s, d, w, vertices, opts, runs=()):
    """the same graph through the single-GPU constructor: {key: {vertex id: value}} as mg_run"""
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import make_graph
    wdt = np.float32 if w is None else w.dtype.type
    h, g = make_graph(s, d, w, store_transposed=True, vertices=vertices, weight_dtype=wdt, **opts)
    out = {}
    v, din, dout = plc.degrees(h, g, None, False)
    out["in"] = dict(zip(v.cpu().tolist(), din.cpu().numpy()))
    out["out"] = dict(zip(v.cpu().tolist(), dout.cpu().numpy()))
    for name, args in runs:
        if name == "pagerank":
            v, x, _ = plc.pagerank(h, g, None, None, None, None, args["alpha"], args["epsilon"], args["max_iterations"], False,
                                   fail_on_nonconvergence=False)
        elif name == "bfs":
            src = torch.as_tensor(np.array([args["source"]], np.int32)).cuda()
            x, _, v = plc.bfs(h, g, src, False, -1, False, False)
        elif name == "sssp":
            v, x, _ = plc.sssp(h, g, args["source"], np.inf, False, False)
        elif name == "wcc":
            v, x = plc.weakly_connected_components(h, g, None, None, None, None, False)
        elif name == "katz":
            v, x = plc.katz_centrality(h, g, None, args["alpha"], 1.0, args["epsilon"], args["max_iterations"], False)
        elif name == "eigenvector":
            v, x = plc.eigenvector_centrality(h, g, args["epsilon"], args["max_iterations"], False)
        elif name == "hits":
            v, hb, au = plc.hits(h, g, args["epsilon"], args["max_iterations"], None, None, True, False)
            out[("hits_auth", "")] = dict(zip(v.cpu().tolist(), au.cpu().numpy()))
            x = hb
        key = (name, str(args)) if name in ("pagerank", "bfs", "sssp") else (name, "")
        out[key] = dict(zip(v.cpu().tolist(), x.cpu().numpy()))
    return out


def same_partition(a, b):
    keys = sorted(a)
    x, y = [a[k] for k in keys], [b[k] for k in keys]
    return len(set(zip(x, y))) == len(set(x)) == len(set(y))


def compare(mg, sg, exact=(), rel=None, partition=()):
    """mg and sg have the same vertices for every key; `exact` keys bit-equal, `rel` {key: tolerance}, `partition` keys the
    same partition"""
    for key in sg:
        assert set(mg[key]) == set(sg[key]), key
        if key in ("in", "out") or key[0] in exact:
            assert all(mg[key][v] == sg[key][v] for v in sg[key]), key
        elif key[0] in partition:
            assert same_partition(mg[key], sg[key]), key
        else:
            tol = rel[key[0]]
            a = np.array([mg[key][v] for v in sorted(sg[key])], np.float64)
            b = np.array([sg[key][v] for v in sorted(sg[key])], np.float64)
            assert np.allclose(a, b, rtol=tol, atol=tol * np.abs(b).max()), (key, np.abs(a - b).max())


# ------------------------------------------------------------------------------------------------ graphs
def hand_graph():
    """self-loops (one a vertex's only edge), multi-edges with distinct and equal weights listed in ascending weight, reverse
    pairs with more copies one way than the other, one-direction edges, and ids 40..44 that no edge touches"""
    e = [(0, 1, 4.0), (0, 1, 5.0), (1, 0, 1.0),             # 2 vs 1 copies: (4 + 1) / 2 and 5
         (1, 2, 3.0), (1, 2, 3.0), (2, 1, 3.0), (2, 1, 7.0),
         (2, 3, 0.5), (3, 4, 2.0), (4, 0, 9.0), (0, 4, 1.0), (0, 4, 2.0),
         (5, 5, 1.0), (5, 6, 1.5), (6, 6, 0.25), (6, 6, 2.0),
         (7, 7, 3.0),                                        # vertex 7: a self-loop only
         (8, 9, 0.75), (9, 10, 0.75), (10, 8, 6.0), (8, 10, 0.125)]
    s = np.array([x[0] for x in e], np.int32)
    d = np.array([x[1] for x in e], np.int32)
    w = np.array([x[2] for x in e], np.float64)
    return s, d, w, np.arange(40, 45, dtype=np.int32)


def rmat_graph(scale, seed=1200, wdtype=np.float32):
    """one-direction RMAT with its duplicates ordered by ascending weight (so that single GPU's first copy is the minimum) and
    self-loops; weights k / 8 so that averages and minima decide shortest paths"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 8 << scale, seed=seed + scale)
    s, d = np.asarray(s, np.int64), np.asarray(d, np.int64)
    rng = np.random.default_rng(seed)
    w = (rng.integers(1, 64, s.size) / 8).astype(wdtype)
    order = np.lexsort((w, d, s))
    return s[order].astype(np.int32), d[order].astype(np.int32), w[order], 1 << scale
