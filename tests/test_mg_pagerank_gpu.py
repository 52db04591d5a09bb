"""Multi-GPU PageRank with personalization, an initial guess and precomputed out-weights on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.pagerank: grids 1x2,
  2x1, 2x2 and 4x2 on directed RMAT-14 and RMAT-16, float32 and float64, against the fp64 oracle and against single-GPU
  personalized PageRank with the same personalization at equal iteration count, on the vertices that appear in edges;
  converging runs within one iteration of single GPU's.
- A world-size-1 NCCL process group running MGGraph.pagerank (the 1x1 grid): the real collectives and the real stream
  ordering on the device.
- 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_centrality_ref as graphs  # noqa: E402
from tests import mg_pagerank_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.test_mg_pagerank_cpu import ITERS, _gloo_graph, _gloo_worker, check_all, check_gloo  # noqa: E402

pytestmark = pytest.mark.gpu


def _converging_runs_match_single_gpu(s, d, V, world):
    """iteration counts at epsilon 1e-6 within one of single GPU's, plain and personalized"""
    import ctypes as C

    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.mg import _views
    from tests.gpu_util import make_graph
    ids, remap = mg_world.present(s, d, V)
    rs, rd, n = remap[s], remap[d], ids.size
    pv = refs.cases(s, d, V)["share_with_zeros"][ids]
    runs = [dict(epsilon=1e-6, max_iterations=500), dict(epsilon=1e-6, max_iterations=500, personalization=(ids, pv))]
    (_, it_plain, conv_plain), (_, it_pers, conv_pers) = refs.mg_pagerank(s, d, V, world, runs, device="cuda")
    h, g = make_graph(rs, rd, store_transposed=True, vertices=np.arange(n, dtype=np.int32))
    L, err = _capi.lib(), C.c_void_p()
    nz = np.flatnonzero(pv != 0).astype(np.int32)
    pids, pvals = torch.as_tensor(nz).cuda(), torch.as_tensor(pv[nz].astype(np.float32)).cuda()
    iters = []
    with _views(pids, pvals) as (vi, vv):
        for name, pers in (("cugraph_pagerank_allow_nonconvergence", []),
                           ("cugraph_personalized_pagerank_allow_nonconvergence", [vi.ptr, vv.ptr])):
            res = C.c_void_p()
            _capi.check(getattr(L, name)(h.ptr, g.ptr, None, None, None, None, *pers, 0.85, 1e-6, 500, 0, C.byref(res),
                                         C.byref(err)), err, name)
            assert L.cugraph_centrality_result_converged(res)
            iters.append(L.cugraph_centrality_result_get_num_iterations(res))
            L.cugraph_centrality_result_free(res)
    torch.cuda.synchronize()
    assert conv_plain and conv_pers
    assert abs(it_plain - iters[0]) <= 1 and abs(it_pers - iters[1]) <= 1, (it_plain, it_pers, iters)


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_pagerank_simulated_on_one_gpu(monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    for scale in (14, 16):
        s, d, V = graphs.rmat_graph(scale)
        check_all(s, d, V, world, device="cuda", single=True)
        _converging_runs_match_single_gpu(s, d, V, world)
    check_all(*graphs.odd_graph(), world, device="cuda", single=True)


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_pagerank_weighted_on_one_gpu(monkeypatch, wdtype):
    s, d, V = graphs.rmat_graph(14)
    w = np.random.default_rng(2).uniform(0.5, 1.0, s.size).astype(wdtype)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), w=w, dtype=wdtype, device="cuda", single=True)


def test_mg_pagerank_float64_rmat16_on_one_gpu(monkeypatch):
    s, d, V = graphs.rmat_graph(16)
    w = np.random.default_rng(3).uniform(0.5, 1.0, s.size)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 4, 2), w=w, dtype=np.float64, device="cuda", single=True)


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _run_nccl(world, golden):
    res = mg_procs.run(_gloo_worker, world, golden["c_api"], "cuda", backend="nccl", timeout=600)
    ids, s, d, V = _gloo_graph()
    check_gloo(res, ids, s, d, V, golden["c_api"], refs.F32_TOL)
    assert ITERS == res[0]["plain"][2]


def test_mg_pagerank_nccl_world_size_1(golden):
    _run_nccl(1, golden)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_pagerank_multi_gpu(world, golden):
    _run_nccl(world, golden)
