"""Multi-GPU SSSP with every rank in ONE process: all P = R x C ranks of a 2D edge partition run through the real block entry
points (cugraph_b200_block_create / _block_sssp_relax / _block_sssp_pred) and the real owner step (mg.sssp_owner_step); the
all-gathers and MIN reduce-scatters between them are tensor ops on one device.  Torch CPU tensors with the emulated library
(tests/emu_py.py) or CUDA tensors with the real one.  The partition is built as in tests/test_emu_mg_cpu.py: edge (u -> v)
lives on rank (r(v), c(u)), row slot c(v) * maxpart + lid(v), column slot r(u) * maxpart + lid(u).

Shared by tests/test_mg_sssp_cpu.py and tests/test_mg_sssp_gpu.py, together with the checks below."""
import ctypes as C
import math

import numpy as np

import oracle


def simulate(s, d, w, V, R, Cc, source, cutoff=math.inf, predecessors=True, delta=None, device="cpu"):
    """Returns (distances [V] in w's dtype, predecessors [V] int64 (-1 = none) or None, stats) indexed by vertex id"""
    import torch
    from cugraph_b200 import _capi, mg
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    P = R * Cc
    dt = torch.float32 if w.dtype == np.float32 else torch.float64
    # vertex -> owner rank, local id inside the owner
    owner = (np.arange(V, dtype=np.int64) * 2654435761 >> 7) % P
    order = np.argsort(owner, kind="stable")
    counts = np.bincount(owner, minlength=P)
    mp = int(counts.max())
    lid = np.empty(V, dtype=np.int64)
    lid[order] = np.arange(V) - np.repeat(np.cumsum(counts) - counts, counts)
    own = [np.where(owner == p)[0][np.argsort(lid[owner == p])] for p in range(P)]
    r_of, c_of = owner // Cc, owner % Cc
    n_rows, n_cols = Cc * mp, R * mp
    handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
    err = C.c_void_p()

    def t(a, dtype=None):
        return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype).to(device)

    blocks, keep = {}, []
    for r in range(R):
        for c in range(Cc):
            m = (r_of[d] == r) & (c_of[s] == c)
            rows = t((c_of[d[m]] * mp + lid[d[m]]).astype(np.int32))
            cols = t((r_of[s[m]] * mp + lid[s[m]]).astype(np.int32))
            ww = t(w[m])
            views = [View(rows), View(cols), View(ww)]
            blk = C.c_void_p()
            code = L.cugraph_b200_block_create(handle.ptr, n_rows, n_cols, views[0].ptr, views[1].ptr, views[2].ptr,
                                               C.byref(blk), C.byref(err))
            _capi.check(code, err, "cugraph_b200_block_create")
            keep.append((rows, cols, ww, views))
            blocks[(r, c)] = blk.value
    if delta is None:
        delta = 32.0 * float(np.mean(w.astype(np.float64))) / (s.size / V) / 64.0
    inf = torch.tensor(math.inf, dtype=dt).to(device)
    big = torch.finfo(dt).max
    dist_own = [torch.full((mp,), big, dtype=dt).to(device) for _ in range(P)]
    pred_code = [torch.full((mp,), -1, dtype=torch.int64).to(device) for _ in range(P)]
    pending = [torch.zeros(mp, dtype=torch.bool).to(device) for _ in range(P)]
    dist_own[owner[source]][lid[source]] = 0
    pending[owner[source]][lid[source]] = True
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
        cand = {}
        x_cols = {}
        for r in range(R):
            for c in range(Cc):
                xc = torch.cat([x[rr * Cc + c] for rr in range(R)])     # all-gather inside the column group
                out = torch.empty(n_rows, dtype=torch.int64).to(device)
                vx, vo = View(xc), View(out)
                code = L.cugraph_b200_block_sssp_relax(handle.ptr, blocks[(r, c)], vx.ptr, float(cutoff), mp, Cc, c, vo.ptr,
                                                       C.byref(err))
                _capi.check(code, err, "cugraph_b200_block_sssp_relax")
                vx.free()
                vo.free()
                cand[(r, c)], x_cols[(r, c)] = out, xc
        improved = [None] * P
        for r in range(R):                                            # MIN reduce-scatter inside the row group
            total = torch.stack([cand[(r, c)] for c in range(Cc)]).min(0).values
            for j in range(Cc):
                p = r * Cc + j
                improved[p] = mg.sssp_owner_step(dist_own[p], pred_code[p], pending[p], total[j * mp:(j + 1) * mp].clone())
        if want_codes:
            win = [torch.where(improved[p], dist_own[p], inf) for p in range(P)]
            for r in range(R):
                codes = []
                for c in range(Cc):
                    wr = torch.cat([win[r * Cc + j] for j in range(Cc)])   # all-gather inside the row group
                    out = torch.empty(n_rows, dtype=torch.int64).to(device)
                    vx, vw, vo = View(x_cols[(r, c)]), View(wr), View(out)
                    code = L.cugraph_b200_block_sssp_pred(handle.ptr, blocks[(r, c)], vx.ptr, vw.ptr, mp, Cc, c, vo.ptr,
                                                          C.byref(err))
                    _capi.check(code, err, "cugraph_b200_block_sssp_pred")
                    for v in (vx, vw, vo):
                        v.free()
                    codes.append(out)
                total = torch.stack(codes).min(0).values
                for j in range(Cc):
                    p = r * Cc + j
                    pred_code[p].copy_(torch.where(improved[p], total[j * mp:(j + 1) * mp], pred_code[p]))
        rounds += 1
    for blk in blocks.values():
        L.cugraph_b200_block_free(blk)
    for *_, views in keep:
        for v in views:
            v.free()
    dist_g = np.empty(V, dtype=w.dtype)
    pred_g = np.full(V, -1, dtype=np.int64)
    for p in range(P):
        dist_g[own[p]] = dist_own[p][:counts[p]].cpu().numpy()
        codes = pred_code[p][:counts[p]].cpu().numpy()
        has = codes >= 0
        pred_g[own[p][has]] = [own[int(k) // mp][int(k) % mp] for k in codes[has]]
    return dist_g, (pred_g if predecessors else None), dict(rounds=rounds, windows=windows)


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
