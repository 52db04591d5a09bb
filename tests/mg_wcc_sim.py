"""Multi-GPU weakly connected components with every rank in ONE process (tests/mg_grid.py): the real block entry point
(cugraph_b200_block_wcc_min) and the real owner step (mg.wcc_owner_step) in the rounds of
MGGraph.weakly_connected_components.

Shared by tests/test_mg_wcc_cpu.py and tests/test_mg_wcc_gpu.py, together with the graphs and checks below."""
import numpy as np

import oracle
from tests.mg_grid import Grid


def simulate(s, d, V, R, Cc, w=None, device="cpu"):
    """Returns (labels [V] int64: the vertex id each vertex's label code names, stats) indexed by vertex id"""
    import torch
    from cugraph_b200 import mg
    grid = Grid(s, d, V, R, Cc, w=w, device=device)
    try:
        P, mp = grid.P, grid.mp
        label_own, changed = [], []
        for p in range(P):
            lab = np.full(mp, mg.INT64_MAX, dtype=np.int64)
            lab[:grid.counts[p]] = p * mp + np.arange(grid.counts[p])
            label_own.append(grid.t(lab))
            changed.append(grid.t(np.arange(mp) < grid.counts[p]))
        rounds = 0
        while True:
            x = [torch.where(changed[p], label_own[p], mg.INT64_MAX) for p in range(P)]
            cand = {}
            for (r, c), blk in grid.blocks.items():
                cand[(r, c)] = torch.empty(grid.n_rows, dtype=torch.int64).to(device)
                grid.call("cugraph_b200_block_wcc_min", blk, grid.gather(x, r, c), cand[(r, c)])
            cand_own = grid.reduce_scatter(cand, op="min")
            changed = [mg.wcc_owner_step(label_own[p], cand_own[p]) for p in range(P)]
            rounds += 1
            if sum(int(ch.sum()) for ch in changed) == 0:
                break
        labels = grid.vertex_of(grid.by_vertex(label_own, dtype=np.int64))
        return labels, dict(rounds=rounds, empty_blocks=grid.empty_blocks)
    finally:
        grid.free()


def single_gpu_wcc(s, d, V):
    """cugraph_weakly_connected_components on the same graph (symmetric, every id 0..V-1 a vertex): labels by vertex id"""
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import by_vertex, make_graph
    h, g = make_graph(s, d, symmetric=True, vertices=np.arange(V, dtype=np.int32))
    verts, labels = plc.weakly_connected_components(h, g, None, None, None, None, False)
    return by_vertex(verts, labels, V)


def same_partition(a, b):
    """the labellings a and b (indexed by vertex) split the vertices into the same sets"""
    return len(set(zip(a.tolist(), b.tolist()))) == len(set(a.tolist())) == len(set(b.tolist()))


def check(s, d, V, labels, single=None):
    """the partition of `labels` is the oracle's (and single-GPU WCC's when given); every label is a vertex of its own
    component, and that vertex carries its own label"""
    ref = oracle.wcc(s, d, V)
    assert labels.shape == (V,)
    assert same_partition(labels, ref)
    if single is not None:
        assert same_partition(labels, single)
    assert ((labels >= 0) & (labels < V)).all()
    assert np.array_equal(ref[labels], ref)
    assert np.array_equal(labels[labels], labels)


def components_graph(seed=5):
    """symmetrised: a small RMAT, a path of 80 vertices (many rounds), 40 disjoint pairs, a vertex whose only edge is a
    self-loop, a star with 30 leaves, duplicate edges, and a few isolated ids"""
    from oracle.rmat import rmat_edgelist
    rs, rd = rmat_edgelist(7, 8 << 7, seed=seed)
    parts_s, parts_d = [np.asarray(rs, np.int64)], [np.asarray(rd, np.int64)]
    base = 1 << 7
    path = np.arange(base, base + 80)
    parts_s.append(path[:-1])
    parts_d.append(path[1:])
    base += 80
    pairs = base + 2 * np.arange(40)
    parts_s.append(pairs)
    parts_d.append(pairs + 1)
    base += 80
    parts_s.append(np.array([base]))                          # the self-loop
    parts_d.append(np.array([base]))
    base += 1
    parts_s.append(np.full(30, base))                         # the star
    parts_d.append(base + 1 + np.arange(30))
    base += 31
    parts_s.append(np.array([path[3], path[3], pairs[0], base - 1]))   # duplicates of existing edges
    parts_d.append(np.array([path[4], path[4], pairs[0] + 1, base - 31]))
    V = base + 5                                              # the last five ids are isolated
    s = np.concatenate(parts_s)
    d = np.concatenate(parts_d)
    # scatter the ids so that components do not sit in runs of consecutive codes
    perm = np.random.default_rng(seed).permutation(V)
    s, d = perm[s], perm[d]
    return np.concatenate([s, d]).astype(np.int32), np.concatenate([d, s]).astype(np.int32), V, 80


def rmat_graph(scale, seed=800):
    """symmetrised RMAT, ef 16"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed + scale)
    s, d = np.asarray(s, np.int32), np.asarray(d, np.int32)
    return np.concatenate([s, d]), np.concatenate([d, s]), 1 << scale
