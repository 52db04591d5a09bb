"""Multi-GPU Katz, eigenvector centrality and HITS on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.katz_centrality /
  .eigenvector_centrality / .hits: grids 1x2, 2x1, 2x2 and 4x2 on a directed RMAT-8 and on a graph with isolated ids,
  sources, sinks and duplicate edges, against the oracle and single-GPU cugraph_katz_centrality / _eigenvector_centrality /
  cugraph_hits on the vertices that appear in edges; a tiny graph that leaves blocks without edges; weighted float32 /
  float64 blocks (float64: the oracle's iteration count, rtol 1e-9) and 64-bit-offset blocks; HITS from an initial
  guess; non-convergence on every rank.
- The owner-step entry points' error paths.
- World sizes 2, 4 and 8 over gloo running the same drivers (the real process groups), with an initial guess given by
  ranks that do not own those vertices and the non-convergence error on every rank."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle  # noqa: E402
from tests import mg_centrality_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]
KATZ_RTOL = 2e-5
EIG_TOL = dict(rtol=2e-3, atol=1e-8)
HITS_TOL = dict(rtol=2e-3, atol=1e-9)


def check_all(s, d, V, world, w=None, dtype=np.float32, device="cpu", single=True):
    """the three algorithms on one grid against the oracle (and single GPU for float32), all on the vertices that appear
    in edges; returns the number of ranks whose block has no edges"""
    ids, remap = mg_world.present(s, d, V)
    rs, rd, n = remap[s], remap[d], ids.size
    f64 = dtype == np.float64
    alpha = refs.katz_alpha(d, V) * (0.5 if w is not None else 1.0)
    runs = [("katz", dict(alpha=alpha, epsilon=1e-6, max_iterations=200)),
            ("eigenvector", dict(epsilon=1e-6, max_iterations=500)), ("hits", dict(epsilon=1e-6, max_iterations=500))]
    got, empty = refs.mg_centrality(s, d, V, world, runs, w=w, dtype=dtype, device=device)
    assert not any(isinstance(r, str) for r in got), got                # an error message
    (katz, kst), (eig, est), (hb, au, hst) = got

    got, it = katz[ids], kst["iterations"]
    want, it_ref = oracle.katz(rs, rd, n, w, alpha=alpha, epsilon=1e-6, dtype=dtype)
    if f64:
        assert it == it_ref
        np.testing.assert_allclose(got, want, rtol=1e-9)
    else:
        np.testing.assert_allclose(got, want, rtol=KATZ_RTOL)
    if single:
        sg, _ = refs.single_gpu("katz", rs, rd, n, w=w, alpha=alpha, epsilon=1e-6, max_iterations=200)
        np.testing.assert_allclose(got, sg, rtol=KATZ_RTOL)

    got, it = eig[ids], est["iterations"]
    want, it_ref = oracle.eigenvector(rs, rd, n, w, epsilon=1e-6)
    if f64:
        assert it == it_ref
        np.testing.assert_allclose(got, want, rtol=1e-9)
    else:
        assert abs(it - it_ref) <= 1
        np.testing.assert_allclose(got, want, **EIG_TOL)
    if single:
        sg, _ = refs.single_gpu("eigenvector", rs, rd, n, w=w, epsilon=1e-6, max_iterations=500)
        np.testing.assert_allclose(got, sg, **EIG_TOL)

    hb, au, it = hb[ids], au[ids], hst["iterations"]
    rh, ra, it_ref, _ = oracle.hits(rs, rd, n, epsilon=1e-6)
    if f64:
        assert it == it_ref
        np.testing.assert_allclose(hb, rh, rtol=1e-9, atol=1e-15)
        np.testing.assert_allclose(au, ra, rtol=1e-9, atol=1e-15)
    else:
        assert abs(it - it_ref) <= 1
        np.testing.assert_allclose(hb, rh, **HITS_TOL)
        np.testing.assert_allclose(au, ra, **HITS_TOL)
    if single:
        sh, sa = refs.single_gpu("hits", rs, rd, n, w=w, epsilon=1e-6, max_iterations=500)
        np.testing.assert_allclose(hb, sh, **HITS_TOL)
        np.testing.assert_allclose(au, sa, **HITS_TOL)
    return empty


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_centrality_simulated_emulated(surface, monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    check_all(*refs.rmat_graph(8), world)
    check_all(*refs.odd_graph(), world)


def test_mg_centrality_empty_blocks_emulated(surface, monkeypatch):
    assert check_all(*refs.tiny_graph(), mg_world.grid_world(monkeypatch, 4, 2), single=False) > 0


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_centrality_weighted_blocks_emulated(surface, monkeypatch, wdtype):
    s, d, V = refs.odd_graph()
    w = np.random.default_rng(2).uniform(0.5, 1.0, s.size).astype(wdtype)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), w=w, dtype=wdtype, single=wdtype == np.float32)


def test_mg_centrality_offs64_emulated(surface, monkeypatch):
    """CUGRAPH_B200_OFFS64_MIN_EDGES=0: the blocks and their column-major copies get 64-bit offsets (the plain sweep)"""
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    s, d, V = refs.rmat_graph(8)
    w = np.random.default_rng(3).uniform(0.5, 1.0, s.size)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), w=w, dtype=np.float64, single=False)


def test_mg_hits_initial_guess_emulated(surface, monkeypatch):
    s, d, V = refs.odd_graph()
    guess = np.random.default_rng(4).uniform(0.0, 2.0, V)
    guess[::3] = 0.0
    ids, remap = mg_world.present(s, d, V)
    runs = [("hits", dict(epsilon=1e-6, max_iterations=500, initial_hubs_guess=(ids, guess[ids])))]
    ((hb, au, st),), _ = refs.mg_centrality(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), runs)
    rh, ra, it_ref, _ = oracle.hits(remap[s], remap[d], ids.size, epsilon=1e-6, initial_hubs=guess[ids])
    assert abs(st["iterations"] - it_ref) <= 1
    np.testing.assert_allclose(hb[ids], rh, **HITS_TOL)
    np.testing.assert_allclose(au[ids], ra, **HITS_TOL)


def test_mg_centrality_nonconvergence_emulated(surface, monkeypatch):
    s, d, V = refs.rmat_graph(8)
    runs = [("katz", dict(alpha=refs.katz_alpha(d, V), epsilon=1e-12, max_iterations=3)),
            ("eigenvector", dict(epsilon=1e-12, max_iterations=3)), ("hits", dict(epsilon=1e-12, max_iterations=3))]
    errors, _ = refs.mg_centrality(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), runs)   # the same on every rank
    for e, msg in zip(errors, ("Katz Centrality", "Eigenvector Centrality", "HITS")):
        assert isinstance(e, str) and f"{msg} failed to converge" in e, e


def test_owner_step_errors_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    handle = ResourceHandle(stream=0)
    part = torch.zeros(2, dtype=torch.float64)
    pp = C.c_void_p(part.data_ptr())
    y, x = torch.ones(8), torch.zeros(8)

    def call(name, *args):
        views = [View(a) if isinstance(a, torch.Tensor) else a for a in args]
        err = C.c_void_p()
        code = getattr(L, name)(handle.ptr, *[v.ptr if isinstance(v, View) else v for v in views], C.byref(err))
        for v in views:
            if isinstance(v, View):
                v.free()
        _capi.check(code, err, name)

    call("cugraph_b200_katz_step", y, x, 8, 0.5, pp)
    assert x.tolist() == [1.5] * 8 and part.tolist() == [12.0, 18.0]
    for args in ((y.double(), x, 8, 0.5, pp), (y, x, 9, 0.5, pp), (y, x, 8, 0.5, None), (y.int(), x.int(), 8, 0.5, pp)):
        with pytest.raises(_capi.CugraphError) as e:
            call("cugraph_b200_katz_step", *args)
        assert e.value.code == _capi.INVALID_INPUT
    with pytest.raises(_capi.CugraphError):
        call("cugraph_b200_hits_scale_step", y, x, x[:4], 8, pp, pp)
    with pytest.raises(_capi.CugraphError):
        call("cugraph_b200_eigenvector_scale_step", y, x, 8, None, pp)
    call("cugraph_b200_katz_step", y[:0], x[:0], 0, 0.5, pp)        # an owner without vertices


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_graph():
    """the odd graph with scattered 64-bit external ids (isolated ids are not vertices of an MG graph)"""
    s, d, V = refs.odd_graph(seed=11)
    ids = np.random.default_rng(11).choice(10**9, size=V, replace=False).astype(np.int64) + 10**10
    return ids, s, d, V


def _guess(ids, s, d):
    present = np.unique(np.concatenate([s, d]))
    vals = np.random.default_rng(5).uniform(0.0, 1.0, present.size)
    return ids[present], vals


def _gloo_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    ids, s, d, V = _gloo_graph()
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    g = mg.MGGraph(torch.from_numpy(ids[s[lo:hi]]), torch.from_numpy(ids[d[lo:hi]]))
    alpha = refs.katz_alpha(d, V)
    out = {}
    v, x = mg.katz_centrality(g, alpha, epsilon=1e-6, max_iterations=200)
    out["katz"] = (v.numpy(), x.numpy(), g.last_katz_stats)
    v, x = mg.eigenvector_centrality(g, epsilon=1e-6, max_iterations=500)
    out["eig"] = (v.numpy(), x.numpy(), g.last_eigenvector_stats)
    v, hb, au = mg.hits(g, epsilon=1e-6, max_iterations=500)
    out["hits"] = (v.numpy(), hb.numpy(), au.numpy(), g.last_hits_stats)
    gv, gx = _guess(ids, s, d)
    mine = slice(None) if rank == world - 1 else slice(0, 0)     # the whole guess from the last rank only
    v, hb, au = mg.hits(g, epsilon=1e-6, max_iterations=500,
                        initial_hubs_guess=(torch.from_numpy(gv[mine]), torch.from_numpy(gx[mine])))
    out["hits_guess"] = (v.numpy(), hb.numpy(), au.numpy(), g.last_hits_stats)
    errs = []
    for call in (lambda: g.katz_centrality(alpha, epsilon=1e-12, max_iterations=2),
                 lambda: g.eigenvector_centrality(epsilon=1e-12, max_iterations=2),
                 lambda: g.hits(epsilon=1e-12, max_iterations=2)):
        try:
            call()
            errs.append(None)
        except RuntimeError as e:
            errs.append(str(e))
    out["errors"] = errs
    bad = torch.from_numpy(gx[:2] - 5.0) if rank == 0 else torch.zeros(0, dtype=torch.float64)
    try:
        g.hits(initial_hubs_guess=(torch.from_numpy(gv[:bad.numel()]), bad))
    except ValueError as e:
        out["negative_guess"] = str(e)
    return out


@pytest.mark.parametrize("world", [2, 4, 8])
def test_mg_centrality_emulated_gloo(world):
    res = mg_procs.run(_gloo_worker, world, emulated=True)
    ids, s, d, V = _gloo_graph()
    present = np.unique(np.concatenate([s, d]))
    k_of = {int(ids[v]): int(v) for v in present}
    # the MG graph has only the vertices that appear in an edge: the oracle runs on that vertex set
    remap = np.full(V, -1)
    remap[present] = np.arange(present.size)
    rs, rd, n = remap[s], remap[d], present.size

    def by_id(key, k):
        out = np.zeros(n)
        cnt = 0
        for r in res:
            v = r[key][0]
            out[remap[[k_of[int(x)] for x in v]]] = r[key][k]
            cnt += v.size
        assert cnt == n
        return out

    alpha = refs.katz_alpha(d, V)
    ref, _ = oracle.katz(rs, rd, n, alpha=alpha, epsilon=1e-6, dtype=np.float32)
    np.testing.assert_allclose(by_id("katz", 1), ref, rtol=KATZ_RTOL)
    ref, _ = oracle.eigenvector(rs, rd, n, epsilon=1e-6)
    np.testing.assert_allclose(by_id("eig", 1), ref, **EIG_TOL)
    rh, ra, _, _ = oracle.hits(rs, rd, n, epsilon=1e-6)
    np.testing.assert_allclose(by_id("hits", 1), rh, **HITS_TOL)
    np.testing.assert_allclose(by_id("hits", 2), ra, **HITS_TOL)
    gv, gx = _guess(ids, s, d)
    init = np.zeros(n)
    init[remap[[k_of[int(x)] for x in gv]]] = gx
    rh, ra, _, _ = oracle.hits(rs, rd, n, epsilon=1e-6, initial_hubs=init)
    np.testing.assert_allclose(by_id("hits_guess", 1), rh, **HITS_TOL)
    np.testing.assert_allclose(by_id("hits_guess", 2), ra, **HITS_TOL)
    for key, k in (("katz", 2), ("eig", 2), ("hits", 3), ("hits_guess", 3)):
        assert all(r[key][k] == res[0][key][k] for r in res)      # every rank ran the same iterations
    for r in res:
        assert len(r["errors"]) == 3 and all(e is not None for e in r["errors"])
        assert "Katz Centrality failed to converge." in r["errors"][0]
        assert "Eigenvector Centrality failed to converge." in r["errors"][1]
        assert "HITS failed to converge." in r["errors"][2]
        assert "initial guess values should be non-negative" in r["negative_guess"]
