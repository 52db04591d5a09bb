"""The WHOLE multi-GPU path on CPU: world_size 2 and 4 processes (gloo), each running cugraph_b200.mg.MGGraph — the real
Python orchestration (2D partition, process groups, all-gather / reduce-scatter / all-to-all, the per-level BFS loop, the
predecessor look-up at the owners) over the real C entry points (cugraph_b200_block_create / _block_pull_sweep /
_pagerank_vertex_step / _block_bfs_pull) of the EMULATED library (tests/emu_py.py: CUDA sources compiled against the SIMT
emulation, torch's CUDA calls given CPU stand-ins).  Results vs the oracle: PageRank at 1e-5 relative (fp32 sweep), BFS
distances exact, BFS predecessors by the reference's validity predicate (cpp/tests/traversal/bfs_test.cpp:213-233).
What this cannot show: NCCL, stream ordering — tests/test_mg_gpu.py does that on 2 / 4 GPUs."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_procs  # noqa: E402


def _graph(V, E, seed):
    rng = np.random.default_rng(seed)
    ids = rng.choice(10**8, size=V, replace=False).astype(np.int64)
    # a hubby graph (sources skewed); a chain entered from the BFS source only, so that BFS has many levels; a few vertices
    # with out-edges only (present, unreachable)
    s_all = (rng.integers(0, V - 100, E) * rng.random(E) ** 2).astype(np.int64)
    d_all = rng.integers(0, V - 100, E)
    chain = np.arange(V - 100, V - 21)
    lonely = np.arange(V - 10, V)
    s_all = np.concatenate([s_all, [s_all[0]], chain, lonely])
    d_all = np.concatenate([d_all, [V - 100], chain + 1, rng.integers(0, V - 100, lonely.size)])
    return ids, s_all, d_all


def _worker(rank, world, V, E):
    from cugraph_b200 import mg
    ids, s_all, d_all = _graph(V, E, 99)
    n = s_all.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    g = mg.MGGraph(torch.from_numpy(ids[s_all[lo:hi]]), torch.from_numpy(ids[d_all[lo:hi]]))
    verts, pr, iters, _ = g.pagerank(alpha=0.85, epsilon=0.0, max_iterations=12)
    bv, bd, bp = g.bfs(int(ids[s_all[0]]))
    return verts.numpy(), pr.numpy(), bv.numpy(), bd.numpy(), bp.numpy()


# grids 2x1, 2x2, 4x2; the last case gives every block 64-bit offsets (the int64_t block sweep and block BFS)
@pytest.mark.parametrize("world,min_edges,offs64_min_edges", [(2, "0", None), (4, "1000000000", None), (8, "0", None), (2, "0", "0")],
                         ids=["2-0", "4-1000000000", "8-0", "2-0-offs64"])
def test_mg_pagerank_and_bfs_emulated_gloo(world, min_edges, offs64_min_edges):
    import oracle
    V, E = 1500, 12000
    env = {"CUGRAPH_B200_SWEEP_MIN_EDGES": min_edges}
    if offs64_min_edges is not None:
        env["CUGRAPH_B200_OFFS64_MIN_EDGES"] = offs64_min_edges
    res = mg_procs.run(_worker, world, V, E, emulated=True, env=env, timeout=600)
    ids, s_all, d_all = _graph(V, E, 99)
    present = np.unique(np.concatenate([s_all, d_all]))
    remap = -np.ones(V, dtype=np.int64)
    remap[present] = np.arange(present.size)
    s, d = remap[s_all], remap[d_all]
    ext = ids[present]
    source = int(ids[s_all[0]])
    # ---- PageRank
    ref, _, _ = oracle.pagerank(s, d, present.size, None, alpha=0.85, epsilon=0.0, max_iterations=12)
    got = {}
    for verts, vals, _, _, _ in res:
        got.update(zip(verts.tolist(), vals.tolist()))
    assert len(got) == present.size
    np.testing.assert_allclose(np.array([got[int(e)] for e in ext]), ref, rtol=1e-5)
    # ---- BFS: distances exact, predecessors valid
    src_k = int(np.flatnonzero(ext == source)[0])
    ref_d, _ = oracle.bfs(s.astype(np.int32), d.astype(np.int32), present.size, np.array([src_k], dtype=np.int32))
    dist_of, pred_of = {}, {}
    for _, _, bv, bd, bp in res:
        dist_of.update(zip(bv.tolist(), bd.tolist()))
        pred_of.update(zip(bv.tolist(), bp.tolist()))
    imax = np.iinfo(np.int32).max
    got_d = np.array([dist_of[int(e)] for e in ext], dtype=np.int64)
    ref_d = np.asarray(ref_d, dtype=np.int64)
    ref_d = np.where((ref_d < 0) | (ref_d >= imax), imax, ref_d)
    assert np.array_equal(got_d, ref_d)
    assert (got_d == imax).any() and got_d[got_d < imax].max() >= 10      # unreachable vertices and a long chain exist
    edges = set(zip(ext[s].tolist(), ext[d].tolist()))
    for e in ext.tolist():
        if e == source or dist_of[e] == imax:
            assert pred_of[e] == -1
        else:
            pe = pred_of[e]
            assert dist_of[pe] == dist_of[e] - 1 and (pe, e) in edges
