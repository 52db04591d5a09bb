"""Multi-GPU strongly connected components on the GPU.

- Every rank of a grid on ONE GPU in one process (tests/mg_world.py) running
  cugraph_b200.mg.MGGraph.strongly_connected_components: grids 1x2, 2x1, 2x2 and 4x2 on the SCC golden cases, the
  reference's multi-GPU C-test graph and directed RMAT-14 and RMAT-16; one graph per phase; both directions of every edge,
  symmetrize=True, listed isolated vertices, self-loops and multi-edges, blocks without edges, 64-bit offsets and weighted
  blocks.  Partition = Tarjan's, scipy's and single-GPU cugraph_strongly_connected_components'; every label a member of its
  own SCC that carries its own label.
- cugraph_b200_block_scc_push against numpy on the device, and its error paths.
- A world-size-1 NCCL process group (the 1x1 grid: the real collectives and stream ordering), and 2 and 4 GPUs over NCCL
  (skipped when fewer GPUs are visible); last_scc_stats the same on every rank."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_scc_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("R,Cc", [(1, 2), (2, 1), (2, 2), (4, 2)], ids=["1x2", "2x1", "2x2", "4x2"])
def test_mg_scc_simulated_on_one_gpu(monkeypatch, R, Cc):
    refs.check_grid(mg_world.grid_world(monkeypatch, R, Cc), "cuda", [14, 16])


def test_mg_scc_phases_on_one_gpu(monkeypatch):
    refs.check_phases(mg_world.grid_world(monkeypatch, 2, 2), "cuda", 400, 40, 5)


def test_mg_scc_edge_cases_on_one_gpu(monkeypatch):
    refs.check_edge_cases(mg_world.grid_world(monkeypatch, 2, 2), "cuda", 20_000, 30_000, seed=5)
    mg_world.grid_world(monkeypatch, 4, 2)
    refs.check_empty_blocks("cuda")


def test_mg_scc_offs64_on_one_gpu(monkeypatch):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, V = refs.rmat_graph(14)
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    labels, _, _ = refs.mg_scc(s, d, V, world, device="cuda")
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    refs.check(s, d, V, labels, single=refs.single_gpu_scc(s, d, V))


def test_mg_scc_weighted_blocks_on_one_gpu(monkeypatch):
    refs.check_weighted(mg_world.grid_world(monkeypatch, 2, 2), "cuda", *refs.rmat_graph(14))


def test_block_scc_push_against_numpy_on_gpu():
    refs.check_entry_point("cuda")
    refs.check_entry_errors("cuda")


# ------------------------------------------------------------------------------------------------- NCCL process groups
def _graphs():
    return [refs.rmat_graph(14), refs.cycle_chain(30, 4), refs.c_test_graph()]


def _nccl_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    out = []
    for s, d, V in _graphs():
        E = s.size
        lo, hi = rank * E // world, (rank + 1) * E // world
        g = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda())
        v, lab = mg.strongly_connected_components(g)
        out.append((v.cpu().numpy(), lab.cpu().numpy(), g.last_scc_stats))
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
        refs.check(s, d, V, labels, single=refs.single_gpu_scc(s, d, V))


def test_mg_scc_nccl_world_size_1():
    _run_nccl(1)


@pytest.mark.parametrize("world", [2, 4])
def test_mg_scc_multi_gpu(world):
    _run_nccl(world)
