"""Multi-GPU weakly connected components with every rank in ONE process: all P = R x C ranks of a 2D edge partition run
through the real block entry points (cugraph_b200_block_create / _block_wcc_min) and the real owner step
(mg.wcc_owner_step); the all-gathers and MIN reduce-scatters between them are tensor ops on one device.  Torch CPU tensors
with the emulated library (tests/emu_py.py) or CUDA tensors with the real one.  The partition is the one of
tests/mg_sssp_sim.py: edge (u -> v) lives on rank (r(v), c(u)), row slot c(v) * maxpart + lid(v), column slot
r(u) * maxpart + lid(u); every id 0..V-1 is a vertex.

Shared by tests/test_mg_wcc_cpu.py and tests/test_mg_wcc_gpu.py, together with the graphs and checks below."""
import ctypes as C

import numpy as np

import oracle


def simulate(s, d, V, R, Cc, w=None, device="cpu"):
    """Returns (labels [V] int64: the vertex id each vertex's label code names, stats) indexed by vertex id"""
    import torch
    from cugraph_b200 import _capi, mg
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    P = R * Cc
    owner = (np.arange(V, dtype=np.int64) * 2654435761 >> 7) % P
    order = np.argsort(owner, kind="stable")
    counts = np.bincount(owner, minlength=P)
    mp = int(counts.max())
    lid = np.empty(V, dtype=np.int64)
    lid[order] = np.arange(V) - np.repeat(np.cumsum(counts) - counts, counts)
    own = [np.where(owner == p)[0][np.argsort(lid[owner == p])] for p in range(P)]
    r_of, c_of = owner // Cc, owner % Cc
    n_rows, n_cols = Cc * mp, R * mp
    handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
    err = C.c_void_p()

    def t(a):
        return torch.as_tensor(np.ascontiguousarray(a)).to(device)

    blocks, keep, empty_blocks = {}, [], 0
    for r in range(R):
        for c in range(Cc):
            m = (r_of[d] == r) & (c_of[s] == c)
            empty_blocks += int(not m.any())
            rows = t((c_of[d[m]] * mp + lid[d[m]]).astype(np.int32))
            cols = t((r_of[s[m]] * mp + lid[s[m]]).astype(np.int32))
            ww = t(w[m]) if w is not None else None
            views = [View(rows), View(cols), View(ww)]
            blk = C.c_void_p()
            code = L.cugraph_b200_block_create(handle.ptr, n_rows, n_cols, views[0].ptr, views[1].ptr, views[2].ptr,
                                               C.byref(blk), C.byref(err))
            _capi.check(code, err, "cugraph_b200_block_create")
            keep.append((rows, cols, ww, views))
            blocks[(r, c)] = blk.value
    imax = np.iinfo(np.int64).max
    label_own, changed = [], []
    for p in range(P):
        lab = np.full(mp, imax, dtype=np.int64)
        lab[:counts[p]] = p * mp + np.arange(counts[p])
        label_own.append(t(lab))
        changed.append(t(np.arange(mp) < counts[p]))
    rounds = 0
    while True:
        x = [torch.where(changed[p], label_own[p], mg.INT64_MAX) for p in range(P)]
        cand = {}
        for r in range(R):
            for c in range(Cc):
                xc = torch.cat([x[rr * Cc + c] for rr in range(R)])     # all-gather inside the column group
                out = torch.empty(n_rows, dtype=torch.int64).to(device)
                vx, vo = View(xc), View(out)
                code = L.cugraph_b200_block_wcc_min(handle.ptr, blocks[(r, c)], vx.ptr, vo.ptr, C.byref(err))
                _capi.check(code, err, "cugraph_b200_block_wcc_min")
                vx.free()
                vo.free()
                cand[(r, c)] = out
        for r in range(R):                                            # MIN reduce-scatter inside the row group
            total = torch.stack([cand[(r, c)] for c in range(Cc)]).min(0).values
            for j in range(Cc):
                p = r * Cc + j
                changed[p] = mg.wcc_owner_step(label_own[p], total[j * mp:(j + 1) * mp].clone())
        rounds += 1
        if sum(int(ch.sum()) for ch in changed) == 0:
            break
    for blk in blocks.values():
        L.cugraph_b200_block_free(blk)
    for *_, views in keep:
        for v in views:
            v.free()
    labels = np.empty(V, dtype=np.int64)
    for p in range(P):
        codes = label_own[p][:counts[p]].cpu().numpy()
        labels[own[p]] = [own[int(k) // mp][int(k) % mp] for k in codes]
    return labels, dict(rounds=rounds, empty_blocks=empty_blocks)


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
