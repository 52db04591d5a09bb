"""Multi-GPU weakly connected components on every rank of a grid in ONE process (tests/mg_world.py:
MGGraph.weakly_connected_components itself), the single-GPU reference, the graphs and the checks.

Shared by tests/test_mg_wcc_cpu.py and tests/test_mg_wcc_gpu.py."""
import numpy as np

import oracle
from tests import mg_world


def _worker(rank, world, s, d, w, device):
    g = mg_world.graph(rank, world, s, d, w, np.float32 if w is None else w.dtype, device)
    v, labels = g.weakly_connected_components()
    assert labels.dtype == v.dtype
    return v, labels, g.last_wcc_stats, g.num_edges_local


def mg_wcc(s, d, V, world, w=None, device="cpu"):
    """MGGraph.weakly_connected_components on `world` ranks.  Returns (labels [V] int64: the vertex id each vertex's label
    names, last_wcc_stats, the number of ranks whose block has no edges) indexed by vertex id; ids without edges are not
    vertices of the graph: components of their own"""
    res = mg_world.run(world, _worker, s, d, w, device)
    labels = mg_world.by_id([r[:2] for r in res], V, -1, np.int64)
    absent = labels < 0
    labels[absent] = np.flatnonzero(absent)
    stats = res[0][2]
    assert all(r[2] == stats for r in res)                        # every rank ran the same rounds
    return labels, stats, sum(r[3] == 0 for r in res)


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
