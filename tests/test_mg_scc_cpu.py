"""Multi-GPU strongly connected components on the CPU, over the emulated library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.strongly_connected_components:
  grids 1x2, 2x1, 2x2 and 4x2 on the SCC golden cases (email-Eu-core on the 2x2 grid only), the reference's multi-GPU C-test
  graph and a directed RMAT-8.  Partition = Tarjan's, scipy's and single-GPU SCC's; every label a member of its own SCC
  that carries its own label.
- One graph per phase (chain: trim; cycle: forward-backward; cycles joined one way: colouring; a pivot with FW\\BW and
  BW\\FW both non-empty), with last_scc_stats showing the phase's rounds.
- Both directions of every edge (MG WCC's labels), symmetrize=True rejected on every rank, listed isolated vertices,
  self-loops and multi-edges, a tiny graph that leaves blocks empty, 64-bit-offset blocks and push structures, and weighted
  float32 / float64 blocks.
- cugraph_b200_block_scc_push called directly against numpy, and its error paths.
- World sizes 2, 4 and 8 over gloo running MGGraph.strongly_connected_components (the real process groups)."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402
from tests import mg_scc_ref as refs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_scc_simulated_emulated(surface, monkeypatch, R, Cc):
    refs.check_grid(mg_world.grid_world(monkeypatch, R, Cc), "cpu", [8], big_goldens=(R, Cc) == (2, 2))


def test_mg_scc_phases_emulated(surface, monkeypatch):
    refs.check_phases(mg_world.grid_world(monkeypatch, 2, 2), "cpu", 100, 12, 4)


def test_mg_scc_edge_cases_emulated(surface, monkeypatch):
    refs.check_edge_cases(mg_world.grid_world(monkeypatch, 2, 2), "cpu", 300, 500, seed=3)


def test_mg_scc_empty_blocks_emulated(surface, monkeypatch):
    mg_world.grid_world(monkeypatch, 4, 2)
    refs.check_empty_blocks("cpu")


def test_mg_scc_offs64_emulated(surface, monkeypatch):
    """CUGRAPH_B200_OFFS64_MIN_EDGES=0: the blocks, their push copies and their row queues get 64-bit offsets"""
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, V = refs.rmat_graph(8)
    want, _, _ = refs.mg_scc(s, d, V, world)
    monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", "0")
    got, _, _ = refs.mg_scc(s, d, V, world)
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    refs.check(s, d, V, got)
    assert np.array_equal(got, want)


def test_mg_scc_weighted_blocks_emulated(surface, monkeypatch):
    refs.check_weighted(mg_world.grid_world(monkeypatch, 2, 2), "cpu", *refs.rmat_graph(8))


def test_block_scc_push_against_numpy_emulated(surface):
    refs.check_entry_point("cpu")


def test_block_scc_push_errors_emulated(surface):
    refs.check_entry_errors("cpu")


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_graph():
    """a chain, a cycle, cycles joined one way and the split graph side by side, with scattered 64-bit external ids"""
    parts, V = [], 0
    for s, d, n in (refs.chain(30), refs.cycle(20), refs.cycle_chain(6, 3), refs.split_graph()):
        parts.append((s.astype(np.int64) + V, d.astype(np.int64) + V))
        V += n
    s, d = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    ids = np.random.default_rng(9).choice(10**9, size=V, replace=False).astype(np.int64) + 10**10
    return ids, s, d, V


def _gloo_worker(rank, world):
    import torch
    from cugraph_b200 import mg
    ids, s, d, V = _gloo_graph()
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    g = mg.MGGraph(torch.from_numpy(ids[s[lo:hi]]), torch.from_numpy(ids[d[lo:hi]]))
    verts, labels = mg.strongly_connected_components(g)
    return dict(verts=verts.numpy(), labels=labels.numpy(), stats=g.last_scc_stats)


@pytest.mark.parametrize("world", [2, 4, 8])
def test_mg_scc_emulated_gloo(world):
    res = mg_procs.run(_gloo_worker, world, emulated=True)
    ids, s, d, V = _gloo_graph()
    k_of = {int(x): k for k, x in enumerate(ids)}
    labels = np.full(V, -1, dtype=np.int64)
    n = 0
    for r in res:
        assert r["labels"].dtype == np.int64
        labels[[k_of[int(v)] for v in r["verts"]]] = [k_of[int(x)] for x in r["labels"]]
        n += r["verts"].size
    assert n == V
    refs.check(s, d, V, labels)
    stats = [r["stats"] for r in res]
    assert all(st == stats[0] for st in stats)                     # every rank ran the same rounds
    assert stats[0]["trim_rounds"] >= 15 and stats[0]["fw_rounds"] > 0 and stats[0]["outer_rounds"] >= 2, stats[0]
