"""Multi-GPU SSSP on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.sssp: grids 1x2, 2x1, 2x2 and
  4x2, float32 and float64, with and without predecessors, with a cutoff, on 64-bit-offset blocks, and on the zero-weight
  graph.  Distances bit-exact vs the oracle and vs single-GPU cugraph_sssp; predecessors valid and a tree.
- World sizes 2, 4 and 8 over gloo running MGGraph.sssp (the real process groups), on a graph with unreachable vertices
  and a weighted chain that takes many windows, and once with everything in one window.
- The error paths of MGGraph.sssp and of the two C entry points."""
import ctypes as C
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_sssp_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

SCALE = 8


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_sssp_simulated_emulated(surface, monkeypatch, R, Cc, wdtype):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, w, V = refs.rmat_graph(SCALE, wdtype)
    srcs = refs.sources(s, V)
    single = {src: refs.single_gpu_sssp(s, d, w, V, src) for src in srcs}
    reach = single[srcs[-1]][single[srcs[-1]] < np.finfo(wdtype).max]
    co = float(np.quantile(reach, 0.3))
    runs = [(src, math.inf, preds) for src in srcs for preds in (True, False)] + [(srcs[0], co, True)]
    res = refs.mg_sssp(s, d, w, V, world, runs)
    for (src, _, _), (dist, pred, stats) in zip(runs, res[:-1]):
        refs.check(s, d, w, V, src, dist, pred, single=single[src])
        assert stats["windows"] > 1
    dist, pred, _ = res[-1]
    refs.check(s, d, w, V, srcs[0], dist, pred, cutoff=co, single=refs.single_gpu_sssp(s, d, w, V, srcs[0], cutoff=co))


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_sssp_simulated_offs64_emulated(surface, monkeypatch, wdtype):
    """CUGRAPH_B200_OFFS64_MIN_EDGES=0: the blocks and their push copies get 64-bit offsets"""
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    s, d, w, V = refs.rmat_graph(SCALE, wdtype)
    src = refs.sources(s, V)[0]
    (dist, pred, _), = refs.mg_sssp(s, d, w, V, mg_world.grid_world(monkeypatch, 2, 2), [(src, math.inf, True)])
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    refs.check(s, d, w, V, src, dist, pred, single=refs.single_gpu_sssp(s, d, w, V, src))


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_sssp_zero_weights_emulated(surface, monkeypatch, wdtype):
    s, d, w, V = refs.zero_weight_graph(wdtype)
    res = refs.mg_sssp(s, d, w, V, mg_world.grid_world(monkeypatch, 2, 2), [(src, math.inf, True) for src in (0, 7)])
    for src, (dist, pred, _) in zip((0, 7), res):
        refs.check(s, d, w, V, src, dist, pred, single=refs.single_gpu_sssp(s, d, w, V, src))


# ---------------------------------------------------------------------------------------------------- C entry point errors
def _tiny_block(L, handle, wdtype, weighted=True):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View
    rows = torch.tensor([0, 1, 2], dtype=torch.int32)
    cols = torch.tensor([1, 2, 0], dtype=torch.int32)
    w = torch.tensor([0.5, 0.25, 1.0], dtype=torch.float32 if wdtype == np.float32 else torch.float64) if weighted else None
    vr, vc, vw = View(rows), View(cols), View(w)
    blk, err = C.c_void_p(), C.c_void_p()
    _capi.check(L.cugraph_b200_block_create(handle.ptr, 3, 3, vr.ptr, vc.ptr, vw.ptr, C.byref(blk), C.byref(err)), err, "create")
    return blk.value, (rows, cols, w, vr, vc, vw)


def test_block_sssp_entry_errors_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    handle = ResourceHandle(stream=0)
    f32, f64, i64 = torch.float32, torch.float64, torch.int64

    def relax(blk, dist_cols, cand, maxpart=3, grid_cols=1, grid_c=0):
        vd, vc, err = View(dist_cols), View(cand), C.c_void_p()
        code = L.cugraph_b200_block_sssp_relax(handle.ptr, blk, vd.ptr, math.inf, maxpart, grid_cols, grid_c, vc.ptr, C.byref(err))
        _capi.check(code, err, "cugraph_b200_block_sssp_relax")

    def pred(blk, dist_cols, win, codes, maxpart=3):
        vd, vw, vc, err = View(dist_cols), View(win), View(codes), C.c_void_p()
        code = L.cugraph_b200_block_sssp_pred(handle.ptr, blk, vd.ptr, vw.ptr, maxpart, 1, 0, vc.ptr, C.byref(err))
        _capi.check(code, err, "cugraph_b200_block_sssp_pred")

    inf = math.inf
    blk, keep = _tiny_block(L, handle, np.float32)
    x = torch.tensor([0.0, inf, inf], dtype=f32)
    cand = torch.empty(3, dtype=i64)
    relax(blk, x, cand)                                              # the valid call: column 0 reaches row 2 at 1.0
    assert cand[2].item() == (int(np.float32(1.0).view(np.uint32)) << 32) and cand[0].item() == cand[1].item() == 2**63 - 1
    bad = [dict(dist_cols=x.double()), dict(cand=cand.int()), dict(dist_cols=x[:2]), dict(cand=cand[:2]),
           dict(grid_c=1), dict(grid_cols=0), dict(maxpart=0),
           dict(maxpart=2**31, grid_cols=2),                          # codes up to 2^32: do not fit a float key
           dict(maxpart=2**40)]
    for kw in bad:
        args = dict(dist_cols=x, cand=cand)
        args.update(kw)
        with pytest.raises(_capi.CugraphError) as e:
            relax(blk, **args)
        assert e.value.code == _capi.INVALID_INPUT, kw
    relax(blk, x, cand, maxpart=2**31, grid_cols=1)                  # R * C * maxpart = 2^31: fits
    with pytest.raises(_capi.CugraphError) as e:                     # the pred call checks its win_rows too
        pred(blk, x, torch.full((3,), inf, dtype=f64), cand)
    assert e.value.code == _capi.INVALID_INPUT
    with pytest.raises(_capi.CugraphError) as e:
        pred(blk, x, torch.full((2,), inf, dtype=f32), cand)
    assert e.value.code == _capi.INVALID_INPUT
    L.cugraph_b200_block_free(blk)
    # float64: the pred call gives the code of the column whose sum reproduces the accepted distance
    blk, keep = _tiny_block(L, handle, np.float64)
    x = torch.tensor([0.0, inf, inf], dtype=f64)
    relax(blk, x, cand, maxpart=2**40)                               # double keys carry no code: any maxpart
    assert cand[2].item() == int(np.float64(1.0).view(np.int64))
    codes = torch.empty(3, dtype=i64)
    pred(blk, x, torch.tensor([inf, inf, 1.0], dtype=f64), codes)
    assert codes.tolist() == [2**63 - 1, 2**63 - 1, 0]
    L.cugraph_b200_block_free(blk)
    blk, keep = _tiny_block(L, handle, np.float32, weighted=False)
    with pytest.raises(_capi.CugraphError) as e:
        relax(blk, torch.zeros(3, dtype=f32), cand)
    assert e.value.code == _capi.INVALID_INPUT
    L.cugraph_b200_block_free(blk)


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_graph(V, E, seed, wdtype):
    """a hubby graph; a chain of weight-1 edges entered from the source only (its distances need many windows); a few
    vertices with out-edges only (present, unreachable)"""
    rng = np.random.default_rng(seed)
    ids = rng.choice(10**8, size=V, replace=False).astype(np.int64)
    s_all = (rng.integers(0, V - 100, E) * rng.random(E) ** 2).astype(np.int64)
    d_all = rng.integers(0, V - 100, E)
    w_all = rng.random(E)
    chain = np.arange(V - 100, V - 21)
    lonely = np.arange(V - 10, V)
    s_all = np.concatenate([s_all, [s_all[0]], chain, lonely])
    d_all = np.concatenate([d_all, [V - 100], chain + 1, rng.integers(0, V - 100, lonely.size)])
    w_all = np.concatenate([w_all, [0.5], np.ones(chain.size), rng.random(lonely.size)]).astype(wdtype)
    return ids, s_all, d_all, w_all


def _gloo_worker(rank, world, V, E):
    import torch
    from cugraph_b200 import mg
    out = {}
    for wdtype in (np.float32, np.float64):
        ids, s_all, d_all, w_all = _gloo_graph(V, E, 99, wdtype)
        n = s_all.size
        lo, hi = rank * n // world, (rank + 1) * n // world
        src = torch.from_numpy(ids[s_all[lo:hi]])
        dst = torch.from_numpy(ids[d_all[lo:hi]])
        g = mg.MGGraph(src, dst, torch.from_numpy(w_all[lo:hi]))
        source = int(ids[s_all[0]])
        runs = [g.sssp(source), g.sssp(source, compute_predecessors=False), g.sssp(source, cutoff=3.0)]
        stats = g.last_sssp_stats
        out[np.dtype(wdtype).name] = ([tuple(None if a is None else a.numpy() for a in r) for r in runs], stats)
        if wdtype == np.float32:
            errors = []
            try:
                g.sssp(-12345)
            except ValueError as e:
                errors.append(str(e))
            gu = mg.MGGraph(src, dst)
            try:
                mg.sssp(gu, source)
            except ValueError as e:
                errors.append(str(e))
            out["errors"] = errors
            del gu
        del g
    return out


@pytest.mark.parametrize("world,delta_scale", [(2, "1"), (4, "1"), (8, "1"), (2, "1e9")],
                         ids=["2", "4", "8", "2-one-window"])
def test_mg_sssp_emulated_gloo(world, delta_scale):
    import oracle
    from tests.test_paths_gpu import _assert_predecessor_tree
    V, E = 1500, 12000
    res = mg_procs.run(_gloo_worker, world, V, E, emulated=True, env={"CUGRAPH_B200_MG_SSSP_DELTA_SCALE": delta_scale})
    for errors in (r["errors"] for r in res):
        assert errors == ["sssp source -12345 is not a vertex of the graph", "SSSP requires a weighted graph"]
    for wdtype in (np.float32, np.float64):
        ids, s_all, d_all, w_all = _gloo_graph(V, E, 99, wdtype)
        present = np.unique(np.concatenate([s_all, d_all]))
        remap = -np.ones(V, dtype=np.int64)
        remap[present] = np.arange(present.size)
        s, d, ext = remap[s_all], remap[d_all], ids[present]
        k_of = {int(e): k for k, e in enumerate(ext)}
        src_k = int(remap[s_all[0]])
        unreached = np.finfo(wdtype).max
        name = np.dtype(wdtype).name
        stats = [r[name][1] for r in res]
        assert all(st == stats[0] for st in stats)                  # every rank ran the same windows and rounds
        if delta_scale == "1":
            assert stats[0]["windows"] >= 10, stats[0]
        else:
            assert stats[0]["windows"] == 1, stats[0]
        for i, cutoff in enumerate([None, None, 3.0]):
            dist_k = np.full(present.size, np.nan, dtype=wdtype)
            pred_k = np.full(present.size, -7, dtype=np.int64)
            for r in res:
                verts, dd, pp = r[name][0][i]
                kk = np.array([k_of[int(v)] for v in verts], dtype=np.int64)
                dist_k[kk] = dd
                if pp is not None:
                    pred_k[kk] = [k_of[int(x)] if x >= 0 else -1 for x in pp]
            ref, _ = oracle.sssp(s.astype(np.int32), d.astype(np.int32), w_all, present.size, src_k, cutoff=cutoff,
                                 use_float=wdtype == np.float32)
            assert np.array_equal(dist_k.astype(np.float64), ref), (name, i)
            assert (dist_k == unreached).any()
            if i == 1:
                continue
            assert oracle.check_sssp_predecessors(s, d, w_all, present.size, dist_k.astype(np.float64), pred_k, src_k)
            _assert_predecessor_tree(dist_k, pred_k, src_k, unreached)
