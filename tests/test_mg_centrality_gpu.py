"""Multi-GPU Katz, eigenvector centrality and HITS on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.katz_centrality /
  .eigenvector_centrality / .hits: grids 1x2, 2x1, 2x2 and 4x2 on directed RMAT-14 and RMAT-16, against the oracle and
  single-GPU cugraph_katz_centrality / _eigenvector_centrality / cugraph_hits on the vertices that appear in edges
  (iterations within one of single GPU's); weighted float32 / float64 blocks and 64-bit-offset blocks.
- A world-size-1 NCCL process group running the same drivers (the 1x1 grid): the real collectives and the real stream
  ordering on the device.
- 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible)."""
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
from tests.test_mg_centrality_cpu import EIG_TOL, HITS_TOL, KATZ_RTOL, check_all  # noqa: E402

pytestmark = pytest.mark.gpu


def _iterations_match_single_gpu(s, d, V, world):
    """iteration counts within one of single GPU's on the graph's vertices"""
    import torch
    from cugraph_b200 import _capi
    from tests.gpu_util import make_graph
    alpha = refs.katz_alpha(d, V)
    runs = [("katz", dict(alpha=alpha, epsilon=1e-6, max_iterations=200)),
            ("eigenvector", dict(epsilon=1e-6, max_iterations=500)), ("hits", dict(epsilon=1e-6, max_iterations=500))]
    ((_, kst), (_, est), (_, _, hst)), _ = refs.mg_centrality(s, d, V, world, runs, device="cuda")
    it_k, it_e, it_h = kst["iterations"], est["iterations"], hst["iterations"]
    ids, remap = mg_world.present(s, d, V)
    h, g = make_graph(remap[s], remap[d], store_transposed=True, vertices=np.arange(ids.size, dtype=np.int32))
    L, res, err = _capi.lib(), C.c_void_p(), C.c_void_p()
    _capi.check(L.cugraph_katz_centrality(h.ptr, g.ptr, None, alpha, 1.0, 1e-6, 200, 0, C.byref(res), C.byref(err)), err, "katz")
    sg_k = L.cugraph_centrality_result_get_num_iterations(res)
    L.cugraph_centrality_result_free(res)
    _capi.check(L.cugraph_eigenvector_centrality(h.ptr, g.ptr, 1e-6, 500, 0, C.byref(res), C.byref(err)), err, "eig")
    sg_e = L.cugraph_centrality_result_get_num_iterations(res)
    L.cugraph_centrality_result_free(res)
    _capi.check(L.cugraph_hits(h.ptr, g.ptr, 1e-6, 500, None, None, 1, 0, C.byref(res), C.byref(err)), err, "hits")
    sg_h = L.cugraph_hits_result_get_number_of_iterations(res)
    L.cugraph_hits_result_free(res)
    torch.cuda.synchronize()
    assert abs(it_k - sg_k) <= 1 and abs(it_e - sg_e) <= 1 and abs(it_h - sg_h) <= 1, (it_k, sg_k, it_e, sg_e, it_h, sg_h)


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_centrality_simulated_on_one_gpu(monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    for scale in (14, 16):
        s, d, V = refs.rmat_graph(scale)
        check_all(s, d, V, world, device="cuda")
        _iterations_match_single_gpu(s, d, V, world)
    check_all(*refs.odd_graph(), world, device="cuda")


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_centrality_weighted_blocks_on_one_gpu(monkeypatch, wdtype):
    s, d, V = refs.rmat_graph(14)
    w = np.random.default_rng(2).uniform(0.5, 1.0, s.size).astype(wdtype)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), w=w, dtype=wdtype, device="cuda", single=wdtype == np.float32)


def test_mg_centrality_offs64_on_one_gpu(monkeypatch):
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    s, d, V = refs.rmat_graph(14)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), device="cuda", single=False)


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _nccl_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    s, d, V = refs.rmat_graph(14)
    E = s.size
    lo, hi = rank * E // world, (rank + 1) * E // world
    g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda())
    alpha = refs.katz_alpha(d, V)
    out = {}
    v, x = mg.katz_centrality(g, alpha, epsilon=1e-6, max_iterations=200)
    out["katz"] = (v.cpu().numpy(), x.cpu().numpy(), g.last_katz_stats)
    v, x = mg.eigenvector_centrality(g, epsilon=1e-6, max_iterations=500)
    out["eig"] = (v.cpu().numpy(), x.cpu().numpy(), g.last_eigenvector_stats)
    v, hb, au = mg.hits(g, epsilon=1e-6, max_iterations=500)
    out["hits"] = (v.cpu().numpy(), hb.cpu().numpy(), au.cpu().numpy(), g.last_hits_stats)
    try:
        g.hits(epsilon=1e-12, max_iterations=2)
    except RuntimeError as e:
        out["error"] = str(e)
    del g
    return out


def _run_nccl(world):
    res = mg_procs.run(_nccl_worker, world, backend="nccl", timeout=600)
    s, d, V = refs.rmat_graph(14)
    present = np.unique(np.concatenate([s, d]))
    remap = np.full(V, -1)
    remap[present] = np.arange(present.size)
    rs, rd, n = remap[s], remap[d], present.size

    def by_id(key, k):
        out = np.zeros(n)
        for r in res:
            out[remap[r[key][0]]] = r[key][k]
        assert sum(r[key][0].size for r in res) == n
        return out

    ref, _ = oracle.katz(rs, rd, n, alpha=refs.katz_alpha(d, V), epsilon=1e-6, dtype=np.float32)
    np.testing.assert_allclose(by_id("katz", 1), ref, rtol=KATZ_RTOL)
    ref, _ = oracle.eigenvector(rs, rd, n, epsilon=1e-6)
    np.testing.assert_allclose(by_id("eig", 1), ref, **EIG_TOL)
    rh, ra, _, _ = oracle.hits(rs, rd, n, epsilon=1e-6)
    np.testing.assert_allclose(by_id("hits", 1), rh, **HITS_TOL)
    np.testing.assert_allclose(by_id("hits", 2), ra, **HITS_TOL)
    for r in res:
        assert r["katz"][2] == res[0]["katz"][2] and r["hits"][3] == res[0]["hits"][3]
        assert "HITS failed to converge." in r["error"]


def test_mg_centrality_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_centrality_multi_gpu(world):
    _run_nccl(world)
