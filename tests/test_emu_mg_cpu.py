"""The C side of multi-GPU PageRank (mg.cu: cugraph_b200_block_create / _block_sweep / _pagerank_vertex_step) on the CPU: all
P = R x C ranks of a 2D edge partition run cugraph_b200.mg.MGGraph.pagerank in ONE process (tests/mg_world.py) with the
emulated library — every rank's rectangular block goes through the real block functions (binned rows with row_vertex, the
piece layout, the sweep kernels, the fused vertex step) and the real collectives' calls, done by the in-process stand-in.
Result vs the fp64 oracle.  (The gloo side of the collectives is covered by tests/test_mg_partition_cpu.py.)"""
import numpy as np
import pytest

import oracle
from tests import mg_world
from tests.emu_py import surface  # noqa: F401
from tests.test_emu_staging_cpu import make_edges


def _worker(rank, world, s, d, w, iters):
    g = mg_world.graph(rank, world, s, d, w)
    v, x, it, _ = g.pagerank(0.85, 0.0, iters)
    assert it == iters
    return v, x


@pytest.mark.parametrize("R,Cc,weighted,min_edges", [(1, 2, False, "0"), (2, 1, False, "0"), (2, 2, False, "0"), (2, 4, True, "0"),
                                                     (4, 2, True, "0"), (2, 2, False, "1000000000")])
def test_2d_partitioned_pagerank_on_one_cpu(surface, monkeypatch, R, Cc, weighted, min_edges):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", min_edges)
    world = mg_world.grid_world(monkeypatch, R, Cc)
    src, dst, w = make_edges(90_000, 400_000, seed=71 + world, weighted=weighted)
    ids, inv = np.unique(np.concatenate([src, dst]), return_inverse=True)
    s, d = inv[:src.size], inv[src.size:]
    V = ids.size
    iters = 8
    got = mg_world.by_id(mg_world.run(world, _worker, s, d, w, iters), V)
    ref, _, _ = oracle.pagerank(s.astype(np.int32), d.astype(np.int32), V, None if not weighted else w.astype(np.float64),
                                alpha=0.85, epsilon=0.0, max_iterations=iters)
    np.testing.assert_allclose(got, ref, rtol=2e-5, atol=0)
