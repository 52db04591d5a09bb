"""Multi-GPU SSSP on every rank of a grid in ONE process (tests/mg_world.py: MGGraph.sssp itself), the single-GPU
reference, the graphs and the checks.

Shared by tests/test_mg_sssp_cpu.py and tests/test_mg_sssp_gpu.py."""
import math

import numpy as np

import oracle
from tests import mg_world


def _worker(rank, world, s, d, w, runs, device):
    g = mg_world.graph(rank, world, s, d, w, w.dtype, device)
    out = []
    for source, cutoff, predecessors in runs:
        v, dist, pred = g.sssp(source, cutoff, predecessors)
        out.append((v, dist, pred, g.last_sssp_stats))
    return out


def mg_sssp(s, d, w, V, world, runs, device="cpu"):
    """MGGraph.sssp on `world` ranks, one graph for all runs = [(source, cutoff, predecessors)].  Per run: (distances [V]
    in w's dtype, predecessors [V] int64 (-1 = none) or None, last_sssp_stats) indexed by vertex id; ids without edges
    are not vertices of the graph: unreached"""
    res = mg_world.run(world, _worker, s, d, w, runs, device)
    out = []
    for k, (_, _, predecessors) in enumerate(runs):
        dist = mg_world.by_id([r[k][:2] for r in res], V, np.finfo(w.dtype).max, w.dtype)
        assert predecessors or all(r[k][2] is None for r in res)
        pred = mg_world.by_id([(r[k][0], r[k][2]) for r in res], V, -1, np.int64) if predecessors else None
        stats = res[0][k][3]
        assert all(r[k][3] == stats for r in res)                 # every rank ran the same windows and rounds
        out.append((dist, pred, stats))
    return out


def single_gpu_sssp(s, d, w, V, source, cutoff=math.inf):
    """cugraph_sssp on the same graph (symmetric, every id 0..V-1 a vertex): distances indexed by vertex id"""
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import by_vertex, make_graph
    h, g = make_graph(s, d, w, symmetric=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=w.dtype.type)
    verts, dist, _ = plc.sssp(h, g, source, cutoff, False, False)
    return by_vertex(verts, dist, V)


def check(s, d, w, V, source, dist, pred, cutoff=math.inf, single=None):
    """distances bit-exact vs the oracle in the same float type (and vs `single`, the single-GPU result, when given);
    predecessors valid, every chain back to the source; unreached = FLT_MAX / DBL_MAX with predecessor -1"""
    from tests.test_paths_gpu import _assert_predecessor_tree
    use_float = w.dtype == np.float32
    unreached = np.finfo(w.dtype).max
    ref, _ = oracle.sssp(s, d, w, V, source, cutoff=None if math.isinf(cutoff) else cutoff, use_float=use_float)
    case = f"{w.dtype} source={source} cutoff={cutoff}"
    assert dist.dtype == w.dtype
    assert np.array_equal(dist.astype(np.float64), ref), case
    assert (dist == unreached).any() or (ref < unreached).all()
    if single is not None:
        assert np.array_equal(dist, single), case + " vs single-GPU"
    if pred is not None:
        assert oracle.check_sssp_predecessors(s, d, w, V, dist.astype(np.float64), pred, source), case
        _assert_predecessor_tree(dist, pred, source, unreached)


def zero_weight_graph(wdtype):
    """the graph of check_sssp_zero_weights (tests/test_paths_gpu.py): zero-weight edges both ways, a zero-weight cycle and a
    weight absorbed by rounding (1e8 + 1 == 1e8 in float, 1e16 + 1 == 1e16 in double)"""
    r = np.random.default_rng(3)
    V = 4000
    hs = r.integers(0, V, 16000).astype(np.int32)
    hd = r.integers(0, V, 16000).astype(np.int32)
    hw = np.where(r.random(16000) < 0.5, 0.0, r.random(16000))
    big = 1e8 if wdtype == np.float32 else 1e16
    extra = [(6, 7, 0.0), (7, 8, 0.0), (8, 9, 0.0), (9, 7, 0.0), (0, 3990, big), (3990, 3991, 1.0), (3991, 3992, 1.0)]
    hs = np.concatenate([hs, np.array([e[0] for e in extra], np.int32)])
    hd = np.concatenate([hd, np.array([e[1] for e in extra], np.int32)])
    hw = np.concatenate([hw, [e[2] for e in extra]]).astype(wdtype)
    return np.concatenate([hs, hd]), np.concatenate([hd, hs]), np.concatenate([hw, hw]), V


def rmat_graph(scale, wdtype, seed=700):
    """symmetrised RMAT with weights U[0, 1) (the same weight on both directions of an edge)"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed + scale)
    s, d = np.asarray(s, np.int32), np.asarray(d, np.int32)
    w = np.random.default_rng(seed + 1).random(s.size).astype(wdtype)
    return np.concatenate([s, d]), np.concatenate([d, s]), np.concatenate([w, w]), 1 << scale


def sources(s, V):
    """the hub and the last non-isolated vertex"""
    deg = np.bincount(s, minlength=V)
    return [int(deg.argmax()), int(np.flatnonzero(deg > 0)[-1])]
