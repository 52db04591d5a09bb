"""Multi-GPU weakly connected components on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running
  cugraph_b200.mg.MGGraph.weakly_connected_components: grids 1x2, 2x1, 2x2 and 4x2 on symmetrised RMAT-14 and RMAT-16
  and on the components graph, on 64-bit-offset blocks, and on weighted float32 / float64 blocks.
- A world-size-1 NCCL process group running MGGraph.weakly_connected_components (the 1x1 grid): the real collectives and
  the real stream ordering on the device.
- 2 and 4 GPUs over NCCL (skipped when fewer GPUs are visible).
Partition = the oracle's and single-GPU cugraph_weakly_connected_components'; every label a vertex of its own component
that carries its own label."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_wcc_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_wcc_simulated_on_one_gpu(monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    for scale in (14, 16):
        s, d, V = refs.rmat_graph(scale)
        labels, _, _ = refs.mg_wcc(s, d, V, world, device="cuda")
        refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))
    s, d, V, path_len = refs.components_graph()
    labels, stats, _ = refs.mg_wcc(s, d, V, world, device="cuda")
    refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))
    assert stats["rounds"] >= path_len // 2, stats


def test_mg_wcc_simulated_offs64_on_one_gpu(monkeypatch):
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    s, d, V = refs.rmat_graph(14)
    labels, _, _ = refs.mg_wcc(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), device="cuda")
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_wcc_weighted_blocks_on_one_gpu(monkeypatch, wdtype):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, V = refs.rmat_graph(14)
    want, _, _ = refs.mg_wcc(s, d, V, world, device="cuda")
    w = np.random.default_rng(1).random(s.size).astype(wdtype)
    got, _, _ = refs.mg_wcc(s, d, V, world, w=w, device="cuda")
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _graphs():
    s, d, V = refs.rmat_graph(14)
    cs, cd, cV, _ = refs.components_graph()
    return [(s, d, V), (cs, cd, cV)]


def _nccl_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    out = []
    for s, d, V in _graphs():
        E = s.size
        lo, hi = rank * E // world, (rank + 1) * E // world
        g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda())
        v, lab = mg.weakly_connected_components(g)
        out.append((v.cpu().numpy(), lab.cpu().numpy(), g.last_wcc_stats))
        del g
    return out


def _run_nccl(world):
    res = mg_procs.run(_nccl_worker, world, backend="nccl", timeout=600)
    for i, (s, d, V) in enumerate(_graphs()):
        present = np.unique(np.concatenate([s, d]))
        labels = np.arange(V, dtype=np.int64)    # ids that are not vertices of the MG graph: components of their own
        n = 0
        for r in res:
            v, lab, st = r[i]
            assert lab.dtype == v.dtype
            labels[v] = lab
            n += v.size
            assert st == res[0][i][2]                   # every rank ran the same rounds
        assert n == present.size
        refs.check(s, d, V, labels, single=refs.single_gpu_wcc(s, d, V))


def test_mg_wcc_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_wcc_multi_gpu(world):
    _run_nccl(world)
