"""The BFS / SSSP certificate (MGGraph.validate_bfs / validate_sssp), the generator slices and the Graph500 harness
(scripts/graph500.py) on every rank of a grid in ONE process (tests/mg_world.py): the graphs, the runs, the corruptions
the certificate must reject, and the checks.

Shared by tests/test_graph500_cpu.py and tests/test_graph500_gpu.py."""
import math

import numpy as np

from tests import mg_paths_ref, mg_sssp_ref, mg_world

RULES = ("not_vertex", "missing", "duplicate", "bad_value", "root", "unreached", "edge", "tree_edge", "cycle")
IMAX = np.iinfo(np.int32).max


def _tensor(a, device):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a)).to(device)


def _graph(rank, world, s, d, w, vertices, device):
    from cugraph_b200 import mg
    s, d, *rest = mg_world.share(rank, world, s, d, *([] if w is None else [w]))
    vx = None if vertices is None else _tensor(mg_world.share(rank, world, vertices)[0], device)
    return mg.MGGraph(_tensor(s, device), _tensor(d, device), _tensor(rest[0], device) if rest else None, vertices=vx)


def _sources_of(rank, world, src, device):
    """a run's sources for this rank: one id (every rank), or this rank's share of an id list"""
    if isinstance(src, list):
        return _tensor(np.asarray(mg_world.share(rank, world, np.asarray(src, np.int32))[0], np.int32), device)
    return src


def _run(g, run, rank, world, device):
    kind, src, kw = run
    if kind == "bfs":
        srcs = _sources_of(rank, world, src, device)
        v, d, p = g.bfs(srcs, kw.get("depth_limit", -1), direction_optimizing=kw.get("direction_optimizing", False))
        return v, d, p, srcs
    v, d, p = g.sssp(src, kw.get("cutoff", math.inf))
    return v, d, p, src


def _validate(g, run, triple, srcs):
    kind, _, kw = run
    if kind == "bfs":
        return g.validate_bfs(*triple, srcs, kw.get("depth_limit", -1))
    return g.validate_sssp(*triple, srcs, kw.get("cutoff", math.inf))


def _accept_worker(rank, world, s, d, w, vertices, runs, device):
    g = _graph(rank, world, s, d, w, vertices, device)
    out = []
    for run in runs:
        v, dd, pp, srcs = _run(g, run, rank, world, device)
        args = (v.clone(), dd.clone(), pp.clone())
        cert = _validate(g, run, (v, dd, pp), srcs)
        assert all(a.equal(b) for a, b in zip(args, (v, dd, pp)))     # no input modified
        out.append((cert, v.cpu().numpy(), dd.cpu().numpy(), pp.cpu().numpy()))
    return out


def accept(s, d, w, world, runs, vertices=None, device="cpu"):
    """every run = (kind, sources, keywords) on `world` ranks, validated: returns per run the certificate (the same on
    every rank, checked) and every rank's (vertices, distances, predecessors)"""
    res = mg_world.run(world, _accept_worker, s, d, w, vertices, runs, device)
    out = []
    for k, run in enumerate(runs):
        certs = [r[k][0] for r in res]
        assert all(c == certs[0] for c in certs), certs
        out.append((certs[0], [r[k][1:] for r in res]))
    return out


def assert_accepts(cert, run):
    assert cert["ok"] and all(cert[k] == 0 for k in RULES), (run, cert)
    assert cert["edges_from_reached"] > 0, (run, cert)


# ---------------------------------------------------------------------------------------------------- single GPU
def _single_gpu_worker(rank, world, s, d, w, V, results, device):
    import torch
    from cugraph_b200 import mg
    g = mg.MGGraph(_tensor(s, device), _tensor(d, device), _tensor(w, device),
                   vertices=torch.arange(V, dtype=torch.int32).to(device))
    src = results["source"]
    certs = [g.validate_bfs(*results["bfs"], src), g.validate_sssp(*results["sssp"], src)]
    verts, dist, pred = results["sssp"]
    bad = dist.clone()
    bad[verts == src] = 1.0                                            # the source's distance must be 0
    certs.append(g.validate_sssp(verts, bad, pred, src))
    return certs


def single_gpu_certificates(s, d, w, V, source, device="cpu"):
    """cugraph_bfs and cugraph_sssp (with predecessors) on the single-GPU graph of the same edges (every id 0 .. V-1 a
    vertex), validated on the one rank of a 1x1 grid: (bfs, sssp, sssp with the source's distance changed)"""
    import torch
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import make_graph
    h, g = make_graph(s, d, w, symmetric=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=w.dtype.type)
    dist, pred, verts = plc.bfs(h, g, torch.tensor([source], dtype=torch.int32, device="cuda"), False, -1, True, False)
    sv, sd, sp = plc.sssp(h, g, source, math.inf, True, False)
    results = {"bfs": (verts, dist, pred), "sssp": (sv, sd, sp), "source": source}
    return mg_world.run(1, _single_gpu_worker, s, d, w, V, results, device)[0]


# ---------------------------------------------------------------------------------------------------- corruptions
def _corrupt_worker(rank, world, s, d, w, run, parts, edits, device):
    """the run's validation on each rank's part of a valid result after each edit (a list of per-rank parts)"""
    g = _graph(rank, world, s, d, w, None, device)
    srcs = _sources_of(rank, world, run[1], device) if run[0] == "bfs" else run[1]
    out = []
    for edit in edits:
        v, dd, pp = (_tensor(a, device) for a in edit[rank])
        out.append(_validate(g, run, (v, dd, pp), srcs))
    return out


def reject(s, d, w, world, run, parts, edits, device="cpu"):
    """the certificates of the edited results (edits: per-rank (vertices, distances, predecessors) lists), each checked to
    be the same on every rank"""
    res = mg_world.run(world, _corrupt_worker, s, d, w, run, parts, edits, device)
    out = []
    for k in range(len(edits)):
        certs = [r[k] for r in res]
        assert all(c == certs[0] for c in certs), certs
        out.append(certs[0])
    return out


def edit(parts, fn):
    """a copy of the per-rank parts with fn(vertices, distances, predecessors) applied to each rank's arrays (fn returns
    the new arrays)"""
    return [fn(v.copy(), dd.copy(), pp.copy()) for v, dd, pp in parts]


def set_at(vid, dist=None, pred=None):
    """an edit: vertex vid, wherever it is given, gets the distance and / or predecessor"""
    def fn(v, dd, pp):
        at = v == vid
        if dist is not None:
            dd[at] = dist
        if pred is not None:
            pp[at] = pred
        return v, dd, pp
    return fn


def by_id(parts):
    """vertex id -> (distance, predecessor) over all ranks' parts"""
    out = {}
    for v, dd, pp in parts:
        for a, b, c in zip(v.tolist(), dd.tolist(), pp.tolist()):
            out[a] = (b, c)
    return out


def bfs_corruptions(s, d, parts, source):
    """(rule, edit) pairs on a valid single-source BFS result over the symmetric graph of (s, d): each edit breaks the rule"""
    res = by_id(parts)
    adj = {}
    for a, b in zip(s.tolist(), d.tolist()):
        adj.setdefault(a, set()).add(b)
    preds = {p for _, p in res.values() if p >= 0}
    reached = [v for v, (dv, _) in res.items() if dv != IMAX and v != source]
    leaf = next(v for v in reached if v not in preds and res[v][0] >= 2)
    inner = next(v for v in reached if res[v][0] >= 2)
    dl, pl = res[leaf]
    far = next(u for u in reached if res[u][0] == dl - 1 and u not in adj.get(leaf, ()))     # one level up, no edge to leaf
    same = next((u for u in adj[leaf] if u != leaf and res[u][0] == dl), None)
    same = same if same is not None else next(u for u in reached if res[u][0] == dl and u != leaf)
    nbr = next(u for u in adj[source] if u != source)
    non_vertex = max(res) + 1000
    out = [("edge", set_at(leaf, dist=dl + 1)),
           ("tree_edge", set_at(inner, dist=res[inner][0] - 1)),
           ("bad_value", set_at(leaf, dist=-1)),
           ("tree_edge", set_at(leaf, pred=far)),
           ("tree_edge", set_at(leaf, pred=same)),
           ("edge", set_at(leaf, dist=IMAX, pred=-1)),
           ("unreached", set_at(leaf, dist=IMAX)),
           ("root", set_at(source, pred=nbr)),
           ("missing", lambda v, dd, pp: (v[v != leaf], dd[v != leaf], pp[v != leaf])),
           ("duplicate", lambda v, dd, pp: (np.concatenate([v, v[v == leaf]]), np.concatenate([dd, dd[v == leaf]]),
                                            np.concatenate([pp, pp[v == leaf]]))),
           ("not_vertex", lambda v, dd, pp: (np.where(v == leaf, non_vertex, v).astype(v.dtype), dd, pp))]
    return out


def zero_cycle(s, d, w, parts, source):
    """an edit that makes two reached vertices joined by zero-weight edges in both directions each other's predecessor"""
    res = by_id(parts)
    zero = {(a, b) for a, b, x in zip(s.tolist(), d.tolist(), w.tolist()) if x == 0}
    for a, b in sorted(zero):
        if a != b and (b, a) in zero and source not in (a, b) and res.get(a, (None,))[0] is not None \
                and res[a][1] >= 0 and res[b][1] >= 0:
            def fn(v, dd, pp, a=a, b=b):
                pp[v == a] = b
                pp[v == b] = a
                return v, dd, pp
            return fn
    raise AssertionError("no zero-weight edge pair between reached vertices")


# ---------------------------------------------------------------------------------------------------- graphs and runs
def rmat_runs(s, V):
    """the BFS and SSSP runs on a symmetric RMAT graph: top-down, direction-optimising, multi-source, depth-limited;
    SSSP with and without a cutoff"""
    hub, last = mg_sssp_ref.sources(s, V)
    many = [hub, last] + [int(x) for x in np.unique(s)[::97][:6]]
    return [("bfs", hub, {}), ("bfs", last, {"direction_optimizing": True}), ("bfs", many, {}),
            ("bfs", many, {"direction_optimizing": True}), ("bfs", hub, {"depth_limit": 2}),
            ("sssp", hub, {}), ("sssp", last, {"cutoff": 0.35})]


def forced():
    """the forced-predecessor graph of tests/mg_paths_ref.py: BFS from its roots, together and one alone"""
    s, d, roots, _ = mg_paths_ref.forced_graph()
    return s, d, [("bfs", [int(x) for x in roots], {}), ("bfs", int(roots[0]), {"direction_optimizing": True})]
