"""Multi-GPU weakly connected components on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.weakly_connected_components:
  grids 1x2, 2x1, 2x2 and 4x2 on the components graph and a symmetrised RMAT-8, a tiny graph that leaves blocks without
  edges, 64-bit-offset blocks and push copies, and weighted float32 / float64 blocks.  Partition = the oracle's and
  single-GPU WCC's; every label a vertex of its own component that carries its own label.
- cugraph_b200_block_wcc_min called directly against a numpy min: every column active, a few, none.
- World sizes 2, 4 and 8 over gloo running MGGraph.weakly_connected_components (the real process groups).
- The error paths of the entry point."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_wcc_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_wcc_simulated_emulated(surface, monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    s, d, V, path_len = refs.components_graph()
    labels, stats, _ = refs.mg_wcc(s, d, V, world)
    refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))
    assert stats["rounds"] >= path_len // 2, stats
    s, d, V = refs.rmat_graph(8)
    labels, _, _ = refs.mg_wcc(s, d, V, world)
    refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))


def test_mg_wcc_empty_blocks_emulated(surface, monkeypatch):
    """three edges over eight blocks: most ranks' blocks have no edges"""
    s = np.array([0, 1, 5, 9, 9, 2], np.int32)
    d = np.array([1, 0, 9, 5, 2, 9], np.int32)
    V = 12
    labels, _, empty = refs.mg_wcc(s, d, V, mg_world.grid_world(monkeypatch, 4, 2))
    assert empty > 0
    refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))


def test_mg_wcc_simulated_offs64_emulated(surface, monkeypatch):
    """CUGRAPH_B200_OFFS64_MIN_EDGES=0: the blocks and their push copies get 64-bit offsets"""
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    s, d, V, _ = refs.components_graph()
    labels, _, _ = refs.mg_wcc(s, d, V, mg_world.grid_world(monkeypatch, 2, 2))
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_wcc_weighted_blocks_emulated(surface, monkeypatch, wdtype):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, V, _ = refs.components_graph()
    want, _, _ = refs.mg_wcc(s, d, V, world)
    w = np.random.default_rng(1).random(s.size).astype(wdtype)
    got, _, _ = refs.mg_wcc(s, d, V, world, w=w)
    assert np.array_equal(got, want)


# ---------------------------------------------------------------------------------------------------- the entry point
def _block(L, handle, rows, cols, n_rows, n_cols, w=None):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View
    keep = [torch.as_tensor(rows, dtype=torch.int32), torch.as_tensor(cols, dtype=torch.int32),
            None if w is None else torch.as_tensor(w)]
    views = [View(k) for k in keep]
    blk, err = C.c_void_p(), C.c_void_p()
    code = L.cugraph_b200_block_create(handle.ptr, n_rows, n_cols, views[0].ptr, views[1].ptr, views[2].ptr, C.byref(blk),
                                       C.byref(err))
    _capi.check(code, err, "cugraph_b200_block_create")
    return blk.value, (keep, views)


def _wcc_min(L, handle, blk, label_cols, cand):
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import View
    vl, vc, err = View(label_cols), View(cand), C.c_void_p()
    code = L.cugraph_b200_block_wcc_min(handle.ptr, blk, vl.ptr, vc.ptr, C.byref(err))
    vl.free()
    vc.free()
    _capi.check(code, err, "cugraph_b200_block_wcc_min")


def test_block_wcc_min_against_numpy_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    L = _capi.lib()
    rng = np.random.default_rng(4)
    n_rows, n_cols, E = 700, 900, 6000
    rows = np.concatenate([np.full(300, 3), rng.integers(0, n_rows - 50, E - 300)]).astype(np.int32)  # one row of degree >= 300
    cols = np.concatenate([rng.integers(0, n_cols, 300), (rng.integers(0, n_cols, E - 300) * rng.random(E - 300) ** 2)]
                          ).astype(np.int32)
    imax = np.iinfo(np.int64).max

    def numpy_min(label):
        want = np.full(n_rows, imax, dtype=np.int64)
        np.minimum.at(want, rows, label[cols])
        return want

    for offs64 in (False, True):
        if offs64:   # read when the handle is created
            os.environ["CUGRAPH_B200_OFFS64_MIN_EDGES"] = "0"
        try:
            handle = ResourceHandle(stream=0)
            blk, keep = _block(L, handle, rows, cols, n_rows, n_cols)
        finally:
            os.environ.pop("CUGRAPH_B200_OFFS64_MIN_EDGES", None)
        label = rng.integers(0, 1 << 40, n_cols).astype(np.int64)
        cand = torch.full((n_rows,), 7, dtype=torch.int64)
        _wcc_min(L, handle, blk, torch.from_numpy(label), cand)                        # every column active
        assert np.array_equal(cand.numpy(), numpy_min(label))
        few = np.full(n_cols, imax, dtype=np.int64)
        deg = np.bincount(cols, minlength=n_cols)
        act = np.flatnonzero(deg == 1)[:3]
        few[act] = label[act]
        cand = torch.full((n_rows,), 7, dtype=torch.int64)
        _wcc_min(L, handle, blk, torch.from_numpy(few), cand)                          # three edges
        assert np.array_equal(cand.numpy(), numpy_min(few))
        assert (cand.numpy() != imax).sum() == act.size
        cand = torch.full((n_rows,), 7, dtype=torch.int64)
        _wcc_min(L, handle, blk, torch.full((n_cols + 5,), imax, dtype=torch.int64), cand)  # none, a longer array
        assert (cand.numpy() == imax).all()
        L.cugraph_b200_block_free(blk)


def test_block_wcc_entry_errors_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    handle = ResourceHandle(stream=0)
    i64 = torch.int64
    for w in (None, np.array([0.5, 0.25, 1.0], np.float32), np.array([0.5, 0.25, 1.0], np.float64)):
        blk, keep = _block(L, handle, [0, 1, 2], [1, 2, 0], 3, 4, w)
        lab = torch.tensor([10, 11, 12, 13], dtype=i64)
        cand = torch.empty(3, dtype=i64)
        _wcc_min(L, handle, blk, lab, cand)                       # weights are accepted and ignored
        assert cand.tolist() == [11, 12, 10]
        for kw in (dict(label_cols=lab.int()), dict(label_cols=lab.double()), dict(cand=cand.int()),
                   dict(cand=cand.double()), dict(label_cols=lab[:3]), dict(cand=cand[:2])):
            args = dict(label_cols=lab, cand=cand)
            args.update(kw)
            with pytest.raises(_capi.CugraphError) as e:
                _wcc_min(L, handle, blk, **args)
            assert e.value.code == _capi.INVALID_INPUT, kw
        vl, vc, err = View(lab), View(cand), C.c_void_p()
        for a, b, c in ((None, vl.ptr, vc.ptr), (blk, None, vc.ptr), (blk, vl.ptr, None)):
            code = L.cugraph_b200_block_wcc_min(handle.ptr, a, b, c, C.byref(err))
            with pytest.raises(_capi.CugraphError) as e:
                _capi.check(code, err, "cugraph_b200_block_wcc_min")
            assert e.value.code == _capi.INVALID_INPUT
        vl.free()
        vc.free()
        L.cugraph_b200_block_free(blk)


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_graph():
    """the components graph with scattered 64-bit external ids (isolated ids are not vertices of an MG graph)"""
    s, d, V, path_len = refs.components_graph(seed=9)
    ids = np.random.default_rng(9).choice(10**9, size=V, replace=False).astype(np.int64) + 10**10
    return ids, s, d, V, path_len


def _gloo_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    ids, s, d, V, _ = _gloo_graph()
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    g = mg.MGGraph(torch.from_numpy(ids[s[lo:hi]]), torch.from_numpy(ids[d[lo:hi]]))
    verts, labels = mg.weakly_connected_components(g)
    return dict(verts=verts.numpy(), labels=labels.numpy(), stats=g.last_wcc_stats)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_mg_wcc_emulated_gloo(world):
    import oracle
    res = mg_procs.run(_gloo_worker, world, emulated=True)
    ids, s, d, V, path_len = _gloo_graph()
    present = np.unique(np.concatenate([s, d]))
    k_of = {int(ids[v]): int(v) for v in present}
    labels = np.full(V, -1, dtype=np.int64)
    n = 0
    for r in res:
        assert r["labels"].dtype == np.int64
        labels[[k_of[int(v)] for v in r["verts"]]] = [k_of[int(x)] for x in r["labels"]]
        n += r["verts"].size
    assert n == present.size
    ref = oracle.wcc(s, d, V)
    assert refs.same_partition(labels[present], ref[present])
    assert np.array_equal(ref[labels[present]], ref[present])
    assert np.array_equal(labels[labels[present]], labels[present])
    stats = [r["stats"] for r in res]
    assert all(st == stats[0] for st in stats)                     # every rank ran the same rounds
    assert stats[0]["rounds"] >= path_len // 2, stats[0]
