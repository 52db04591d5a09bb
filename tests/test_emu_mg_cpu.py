"""The C side of multi-GPU PageRank (mg.cu: cugraph_b200_block_create / _block_sweep / _pagerank_vertex_step) on the CPU: all
P = R x C ranks of a 2D edge partition are simulated in ONE process (tests/mg_grid.py) with the emulated library — every
rank's rectangular block goes through the real block functions (binned rows with row_vertex, the piece layout, the sweep
kernels, the fused vertex step), the all-gather / reduce-scatter / 2-scalar all-reduce between them are tensor ops.  Result
vs the fp64 oracle.  (The torch.distributed side — partition_edges, the collectives — is covered by
tests/test_mg_partition_cpu.py with gloo.)"""
import numpy as np
import pytest

import oracle
from tests.emu_py import surface  # noqa: F401
from tests.mg_grid import Grid
from tests.test_emu_staging_cpu import make_edges


@pytest.mark.parametrize("R,Cc,weighted,min_edges", [(1, 2, False, "0"), (2, 1, False, "0"), (2, 2, False, "0"), (2, 4, True, "0"),
                                                     (4, 2, True, "0"), (2, 2, False, "1000000000")])
def test_2d_partitioned_pagerank_on_one_cpu(surface, monkeypatch, R, Cc, weighted, min_edges):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", min_edges)
    P = R * Cc
    src, dst, w = make_edges(90_000, 400_000, seed=71 + P, weighted=weighted)
    ids, inv = np.unique(np.concatenate([src, dst]), return_inverse=True)
    s, d = inv[:src.size], inv[src.size:]
    V = ids.size
    grid = Grid(s, d, V, R, Cc, w=w if weighted else None)
    try:
        # out-weight sums of the owned vertices
        ow_global = np.bincount(s, weights=w.astype(np.float64) if weighted else None, minlength=V)
        out_w, pr, x_loc, yred = [], [], [], [grid.zeros(grid.mp) for _ in range(P)]
        for p in range(P):
            n = grid.counts[p]
            out_w.append(grid.zeros(grid.mp))
            out_w[p][:n] = grid.t(ow_global[grid.own[p]].astype(np.float32))
            pr.append(grid.zeros(grid.mp))
            pr[p][:n] = 1.0 / V
            x_loc.append(grid.zeros(grid.mp))
        tot = grid.scalars(2)
        alpha, iters = 0.85, 8

        def vertex_steps(first):
            parts = [grid.scalars(2) for _ in range(P)]
            for p in range(P):
                grid.call("cugraph_b200_pagerank_vertex_step", yred[p], pr[p], out_w[p], x_loc[p], int(grid.counts[p]), alpha,
                          float(V), int(first), tot, parts[p])
            grid.all_reduce(parts)                                     # the 2-element all-reduce
            tot.copy_(parts[0])

        vertex_steps(True)
        for _ in range(iters):
            # the block's y arrays are the same every iteration: from the second sweep on a block only rewrites the rows
            # that have edges
            yred = grid.spmv(x_loc, alpha)
            vertex_steps(False)
        got = grid.by_vertex(pr)
    finally:
        grid.free()
    ref, _, _ = oracle.pagerank(s.astype(np.int32), d.astype(np.int32), V, None if not weighted else w.astype(np.float64),
                                alpha=alpha, epsilon=0.0, max_iterations=iters)
    np.testing.assert_allclose(got, ref, rtol=2e-5, atol=0)
