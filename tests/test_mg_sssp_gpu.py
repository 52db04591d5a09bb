"""Multi-GPU SSSP on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.sssp: grids 1x2,
  2x1, 2x2 and 4x2 on symmetrised weighted RMAT-14 and RMAT-16, float32 and float64, with and without predecessors, a
  cutoff, 64-bit-offset blocks, and the zero-weight graph.
- A world-size-1 NCCL process group running MGGraph.sssp (the 1x1 grid): the real collectives and the real stream
  ordering on the device.
- 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible).
Distances bit-exact vs the oracle in the same float type and vs single-GPU cugraph_sssp; predecessors by the oracle's
predicate and by walking every chain back to the source."""
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

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
@pytest.mark.parametrize("scale", [14, 16])
def test_mg_sssp_simulated_on_one_gpu(monkeypatch, R, Cc, scale):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    for wdtype in (np.float32, np.float64):
        s, d, w, V = refs.rmat_graph(scale, wdtype)
        srcs = refs.sources(s, V)
        single = {src: refs.single_gpu_sssp(s, d, w, V, src) for src in srcs}
        runs = [(src, math.inf, True) for src in srcs]
        if wdtype == np.float32:
            reach = single[srcs[-1]][single[srcs[-1]] < np.finfo(wdtype).max]
            co = float(np.quantile(reach, 0.3))
            runs += [(srcs[0], math.inf, False), (srcs[-1], co, True)]
        res = refs.mg_sssp(s, d, w, V, world, runs, device="cuda")
        for (src, cutoff, _), (dist, pred, _) in zip(runs, res):
            sg = single[src] if math.isinf(cutoff) else refs.single_gpu_sssp(s, d, w, V, src, cutoff=cutoff)
            refs.check(s, d, w, V, src, dist, pred, cutoff=cutoff, single=sg)


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_sssp_simulated_offs64_on_one_gpu(monkeypatch, wdtype):
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    s, d, w, V = refs.rmat_graph(14, wdtype)
    src = refs.sources(s, V)[0]
    (dist, pred, _), = refs.mg_sssp(s, d, w, V, mg_world.grid_world(monkeypatch, 2, 2), [(src, math.inf, True)],
                                   device="cuda")
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    refs.check(s, d, w, V, src, dist, pred, single=refs.single_gpu_sssp(s, d, w, V, src))


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_sssp_zero_weights_on_one_gpu(monkeypatch, wdtype):
    s, d, w, V = refs.zero_weight_graph(wdtype)
    for R, Cc in ((2, 2), (4, 2)):
        res = refs.mg_sssp(s, d, w, V, mg_world.grid_world(monkeypatch, R, Cc), [(src, math.inf, True) for src in (0, 7)],
                          device="cuda")
        for src, (dist, pred, _) in zip((0, 7), res):
            refs.check(s, d, w, V, src, dist, pred, single=refs.single_gpu_sssp(s, d, w, V, src))


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _nccl_worker(rank, world, scale):
    import torch
    from cugraph_b200 import mg
    out = {}
    for wdtype in (np.float32, np.float64):
        s, d, w, V = refs.rmat_graph(scale, wdtype)
        E = s.size
        lo, hi = rank * E // world, (rank + 1) * E // world
        g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda(), torch.as_tensor(w[lo:hi]).cuda())
        srcs = refs.sources(s, V)
        runs = []
        for src in srcs:
            v, dd, pp = g.sssp(src)
            runs.append((src, v.cpu().numpy(), dd.cpu().numpy(), pp.cpu().numpy()))
        out[np.dtype(wdtype).name] = runs
        del g
    return out


def _run_nccl(world, scale):
    res = mg_procs.run(_nccl_worker, world, scale, backend="nccl", timeout=600)
    for wdtype in (np.float32, np.float64):
        s, d, w, V = refs.rmat_graph(scale, wdtype)
        present = np.unique(np.concatenate([s, d]))
        name = np.dtype(wdtype).name
        for i, src in enumerate(refs.sources(s, V)):
            unreached = np.finfo(wdtype).max
            dist = np.full(V, unreached, dtype=wdtype)   # isolated ids are not vertices of the MG graph: unreached
            pred = np.full(V, -1, dtype=np.int64)
            n = 0
            for r in res:
                _, v, dd, pp = r[name][i]
                dist[v] = dd
                pred[v] = pp
                n += v.size
            assert n == present.size
            refs.check(s, d, w, V, src, dist, pred, single=refs.single_gpu_sssp(s, d, w, V, src))


def test_mg_sssp_nccl_world_size_1():
    _run_nccl(1, 14)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_sssp_multi_gpu(world):
    _run_nccl(world, 14)
