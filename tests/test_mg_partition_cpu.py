"""world_size-2 and -4 gloo runs on CPU: the 2D partition / renumbering / exchange logic of
cugraph_b200.mg (the N>1 host path).  The per-block sweep is done here with plain torch ops — the CUDA
kernels are covered by the -m gpu tests; this file checks that the blocks + collectives reproduce the
global graph and the oracle's PageRank (the reference's MG tests compare MG vs SG the same way,
cpp/tests/link_analysis/mg_pagerank_test.cpp:158-248)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402


def _graph(V, E):
    rng = np.random.default_rng(1234)
    ids = rng.choice(10**9, size=V, replace=False).astype(np.int64)      # arbitrary external ids
    return ids, rng.integers(0, V, E), rng.integers(0, V, E), rng.random(E) + 0.25


def _worker(rank, world, V, E, weighted):
    from cugraph_b200 import mg
    ids, s_all, d_all, w_all = _graph(V, E)
    lo, hi = rank * E // world, (rank + 1) * E // world                  # this rank's share of the edge list
    src = torch.from_numpy(ids[s_all[lo:hi]])
    dst = torch.from_numpy(ids[d_all[lo:hi]])
    w = torch.from_numpy(w_all[lo:hi]) if weighted else None
    groups = mg.make_groups()
    part = mg.partition_edges(src, dst, w, groups)
    g = part.groups
    mp_ = part.maxpart
    # ---- every edge landed on the right GPU, with slots that decode back to its external endpoints
    verts = [None] * world
    dist.all_gather_object(verts, part.vertices.numpy())
    r_u = (part.cols.long() // part.maxpart).numpy()
    c_v = (part.rows.long() // mp_).numpy()
    src_owner = r_u * g.C + g.c
    dst_owner = g.r * g.C + c_v
    dec_src = np.array([verts[o][l] for o, l in zip(src_owner, (part.cols.long() % part.maxpart).numpy())], dtype=np.int64)
    dec_dst = np.array([verts[o][l] for o, l in zip(dst_owner, (part.rows.long() % mp_).numpy())], dtype=np.int64)
    block = (dec_src, dec_dst, None if w is None else part.weights.numpy())
    # ---- PageRank with the same iteration structure as MGGraph.pagerank, block sweep in torch
    alpha, iters = 0.85, 25
    ones = part.weights.double() if weighted else torch.ones(part.cols.numel(), dtype=torch.float64)
    partial = torch.zeros(g.R * mp_, dtype=torch.float64).index_add_(0, part.cols.long(), ones)
    out_w = torch.empty(mp_, dtype=torch.float64)
    mg.reduce_scatter_into(out_w, partial, g.col_group)
    pr = torch.zeros(mp_, dtype=torch.float64)
    pr[:part.n_local] = 1.0 / part.n_global
    xg = torch.zeros(g.R * mp_, dtype=torch.float64)
    yred = torch.zeros(mp_, dtype=torch.float64)
    valid = torch.arange(mp_) < part.n_local

    def step(first, dangling_prev):
        nonlocal pr
        init = 0.0 if first else (dangling_prev * alpha + 1 - alpha) / part.n_global
        new = pr.clone() if first else torch.where(valid, yred + init, torch.zeros_like(yred))
        dang = new[valid & (out_w == 0)].sum().reshape(1)
        x = torch.where(out_w == 0, new, new / torch.where(out_w == 0, torch.ones_like(out_w), out_w))
        pr = new
        dist.all_reduce(dang)
        return x, float(dang)

    x, dang = step(True, 0.0)
    for _ in range(iters):
        xseg = torch.zeros(g.R * mp_, dtype=torch.float64)
        mg.all_gather_into(xseg, x, g.col_group)
        xg = xseg   # partition-major columns: the all-gather output is the block's column order
        ypart = torch.zeros(g.C * mp_, dtype=torch.float64).index_add_(0, part.rows.long(), alpha * xg[part.cols.long()] * ones)
        mg.reduce_scatter_into(yred, ypart, g.row_group)
        x, dang = step(False, dang)
    return block, part.vertices.numpy(), pr[:part.n_local].numpy(), part.n_global


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("weighted", [False, True])
def test_partition_and_pagerank_gloo(world, weighted):
    import oracle
    V, E = 300, 4000
    out = mg_procs.run(_worker, world, V, E, weighted, timeout=180)
    blocks = [o[0] for o in out]
    res = [o[1:3] for o in out]
    n_global = out[0][3]
    ids, s_all, d_all, w_all = _graph(V, E)
    # the union of the blocks is exactly the input multigraph
    got = np.concatenate([np.stack([b[0], b[1]], 1) for b in blocks])
    exp = np.stack([ids[s_all], ids[d_all]], 1)
    assert got.shape == exp.shape
    assert np.array_equal(got[np.lexsort((got[:, 1], got[:, 0]))], exp[np.lexsort((exp[:, 1], exp[:, 0]))])
    present = np.unique(np.concatenate([s_all, d_all]))
    assert n_global == present.size
    # MG PageRank == oracle on the gathered graph
    remap = -np.ones(V, dtype=np.int64)
    remap[present] = np.arange(present.size)
    ref, _, _ = oracle.pagerank(remap[s_all], remap[d_all], present.size, w_all if weighted else None, alpha=0.85,
                                epsilon=0.0, max_iterations=25)
    got_pr = {}
    for verts, vals in res:
        got_pr.update(zip(verts.tolist(), vals.tolist()))
    assert len(got_pr) == present.size
    for k, v in enumerate(present):
        assert got_pr[int(ids[v])] == pytest.approx(ref[k], rel=1e-9)


def test_grid_shape_matches_reference(monkeypatch):
    from cugraph_b200 import mg
    # cpp/tests/utilities/mg_utilities.cpp:49-53: the two factors are the largest divisor <= sqrt(P) and its cofactor; the
    # larger one is the all-gather group here (fewer destination rows per block), the reference's orientation is selectable
    assert mg.grid_shape(1) == (1, 1)
    assert mg.grid_shape(2) == (2, 1)
    assert mg.grid_shape(4) == (2, 2)
    assert mg.grid_shape(8) == (4, 2)
    assert mg.grid_shape(6) == (3, 2)
    monkeypatch.setenv("CUGRAPH_B200_MG_GRID", "wide")
    assert mg.grid_shape(2) == (1, 2) and mg.grid_shape(8) == (2, 4) and mg.grid_shape(6) == (2, 3)


def test_vertex_owner_balanced():
    from cugraph_b200 import mg
    ids = torch.arange(0, 1 << 16, dtype=torch.int32)
    o = mg.vertex_owner(ids, 8)
    cnt = torch.bincount(o, minlength=8).double()
    assert o.min() >= 0 and o.max() < 8
    assert (cnt.max() - cnt.min()) / cnt.mean() < 0.05
