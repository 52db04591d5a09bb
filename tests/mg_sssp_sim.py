"""Multi-GPU SSSP with every rank in ONE process (tests/mg_grid.py): the real block entry points (cugraph_b200_block_sssp_relax /
_block_sssp_pred) and the real owner step (mg.sssp_owner_step) in the rounds and windows of MGGraph.sssp.

Shared by tests/test_mg_sssp_cpu.py and tests/test_mg_sssp_gpu.py, together with the checks below."""
import math

import numpy as np

import oracle
from tests.mg_grid import Grid


def simulate(s, d, w, V, R, Cc, source, cutoff=math.inf, predecessors=True, delta=None, device="cpu"):
    """Returns (distances [V] in w's dtype, predecessors [V] int64 (-1 = none) or None, stats) indexed by vertex id"""
    import torch
    from cugraph_b200 import mg
    grid = Grid(s, d, V, R, Cc, w=w, device=device)
    try:
        P, mp, dt = grid.P, grid.mp, grid.tt
        if delta is None:
            delta = 32.0 * float(np.mean(w.astype(np.float64))) / (w.size / grid.V) / 64.0
        inf = torch.tensor(math.inf, dtype=dt).to(device)
        big = torch.finfo(dt).max
        dist_own = [torch.full((mp,), big, dtype=dt).to(device) for _ in range(P)]
        pred_code = [torch.full((mp,), -1, dtype=torch.int64).to(device) for _ in range(P)]
        pending = [torch.zeros(mp, dtype=torch.bool).to(device) for _ in range(P)]
        dist_own[grid.owner[source]][grid.lid[source]] = 0
        pending[grid.owner[source]][grid.lid[source]] = True
        want_codes = predecessors and dt == torch.float64
        hi = mg.window_bound(0.0, delta, dt, device)
        rounds = windows = 0
        while True:
            active = [pending[p] & (dist_own[p] < hi) for p in range(P)]
            if sum(int(a.sum()) for a in active) == 0:
                windows += 1
                lo = min(float(torch.where(pending[p], dist_own[p], inf).min()) for p in range(P))
                if math.isinf(lo):
                    break
                hi = mg.window_bound(lo, delta, dt, device)
                continue
            x = []
            for p in range(P):
                pending[p] &= ~active[p]
                x.append(torch.where(active[p], dist_own[p], inf))
            cand, x_cols = {}, {}
            for (r, c), blk in grid.blocks.items():
                x_cols[(r, c)] = grid.gather(x, r, c)
                cand[(r, c)] = torch.empty(grid.n_rows, dtype=torch.int64).to(device)
                grid.call("cugraph_b200_block_sssp_relax", blk, x_cols[(r, c)], float(cutoff), mp, Cc, c, cand[(r, c)])
            cand_own = grid.reduce_scatter(cand, op="min")
            improved = [mg.sssp_owner_step(dist_own[p], pred_code[p], pending[p], cand_own[p]) for p in range(P)]
            if want_codes:
                win = [torch.where(improved[p], dist_own[p], inf) for p in range(P)]
                codes = {}
                for (r, c), blk in grid.blocks.items():
                    codes[(r, c)] = torch.empty(grid.n_rows, dtype=torch.int64).to(device)
                    grid.call("cugraph_b200_block_sssp_pred", blk, x_cols[(r, c)], grid.gather(win, r, c, rows=True), mp, Cc, c,
                              codes[(r, c)])
                code_own = grid.reduce_scatter(codes, op="min")
                for p in range(P):
                    pred_code[p].copy_(torch.where(improved[p], code_own[p], pred_code[p]))
            rounds += 1
        dist_g = grid.by_vertex(dist_own, dtype=w.dtype)
        pred_g = grid.vertex_of(grid.by_vertex(pred_code, dtype=np.int64))
        return dist_g, (pred_g if predecessors else None), dict(rounds=rounds, windows=windows)
    finally:
        grid.free()


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
