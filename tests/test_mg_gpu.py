"""2- and 4-GPU NCCL run of the multi-GPU PageRank and BFS (skipped when fewer than 2 GPUs are visible): MG result ==
oracle on the gathered graph, as the reference's mg_pagerank_test.cpp:158-248 compares MG with SG."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pytestmark = pytest.mark.gpu

from tests import mg_procs  # noqa: E402


def _worker(rank, world, scale, weighted):
    import torch
    from cugraph_b200 import mg
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=5)
    E = s.shape[0]
    w_all = np.random.default_rng(3).random(E).astype(np.float32) + 0.1
    lo, hi = rank * E // world, (rank + 1) * E // world
    w = torch.as_tensor(w_all[lo:hi]).cuda() if weighted else None
    G = mg.MGGraph(torch.as_tensor(s[lo:hi]).cuda(), torch.as_tensor(d[lo:hi]).cuda(), w)
    verts, pr, iters, conv = G.pagerank(0.85, 0.0, 40)
    # converging run: iteration count must agree on all ranks and with the scalar exchange
    v2, p2, it2, c2 = G.pagerank(0.85, 1e-6, 500)
    bv, bd, bp = G.bfs(int(s[0]))
    return (verts.cpu().numpy(), pr.cpu().numpy()), it2, c2, (bv.cpu().numpy(), bd.cpu().numpy(), bp.cpu().numpy())


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("weighted", [False, True])
def test_mg_pagerank_multi_gpu(weighted, world):
    import oracle
    from oracle.rmat import rmat_edgelist
    scale = 14
    out = mg_procs.run(_worker, world, scale, weighted, backend="nccl", timeout=300)
    res, it2, c2, bres = [o[0] for o in out], out[0][1], out[0][2], [o[3] for o in out]
    s, d = rmat_edgelist(scale, 16 << scale, seed=5)
    w_all = np.random.default_rng(3).random(s.shape[0]).astype(np.float32) + 0.1
    present = np.unique(np.concatenate([s, d]))
    remap = -np.ones(1 << scale, dtype=np.int64)
    remap[present] = np.arange(present.size)
    ref, _, _ = oracle.pagerank(remap[s], remap[d], present.size, w_all if weighted else None, alpha=0.85, epsilon=0.0,
                                max_iterations=40)
    got = np.zeros(present.size)
    n = 0
    for verts, vals in res:
        got[remap[verts]] = vals
        n += verts.size
    assert n == present.size
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=1e-12)
    _, it_ref, conv_ref = oracle.pagerank(remap[s], remap[d], present.size, w_all if weighted else None, alpha=0.85,
                                          epsilon=1e-6, max_iterations=500)
    assert c2 == conv_ref and abs(it2 - it_ref) <= 1
    # multi-GPU BFS: distances bit-exact vs the oracle, predecessors by the reference's predicate (bfs_test.cpp:213-233)
    ref_d, _ = oracle.bfs(remap[s].astype(np.int32), remap[d].astype(np.int32), present.size,
                          np.array([remap[s[0]]], dtype=np.int32))
    imax = np.iinfo(np.int32).max
    ref_d = np.asarray(ref_d, dtype=np.int64)
    ref_d = np.where((ref_d < 0) | (ref_d >= imax), imax, ref_d)
    got_d = np.full(present.size, -5, dtype=np.int64)
    got_p = np.full(present.size, -5, dtype=np.int64)
    for bv, bd, bp in bres:
        got_d[remap[bv]] = bd
        got_p[remap[bv]] = np.where(bp >= 0, remap[np.maximum(bp, 0)], -1)
    assert np.array_equal(got_d, ref_d)
    edges = set(zip(remap[s].tolist(), remap[d].tolist()))
    for v in np.flatnonzero((ref_d < imax) & (ref_d > 0))[:20000]:
        pv = int(got_p[v])
        assert pv >= 0 and ref_d[pv] == ref_d[v] - 1 and (pv, int(v)) in edges
    assert got_p[remap[s[0]]] == -1 and (got_p[ref_d == imax] == -1).all()
