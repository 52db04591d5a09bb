"""Multi-GPU Katz, eigenvector centrality and HITS with every rank in ONE process: all P = R x C ranks of a 2D edge partition
run through the real block entry points (cugraph_b200_block_create / _block_sweep, pull and transposed) and the real owner
steps (cugraph_b200_katz_step, _eigenvector_add_step / _scale_step, _hits_max_step / _scale_step, _vertex_sum / _scale);
the all-gathers, reduce-scatters and all-reduces between them are tensor ops on one device, in the groups MGGraph uses:
a pull sweep gathers x in the column group and reduces y in the row group, a transposed sweep the other way round.  Torch
CPU tensors with the emulated library (tests/emu_py.py) or CUDA tensors with the real one.  The partition is the one of
tests/mg_wcc_sim.py: edge (u -> v) lives on rank (r(v), c(u)), row slot c(v) * maxpart + lid(v), column slot
r(u) * maxpart + lid(u); every id 0..V-1 is a vertex.

Shared by tests/test_mg_centrality_cpu.py and tests/test_mg_centrality_gpu.py, together with the graphs and checks below."""
import ctypes as C

import numpy as np

F32, F64 = 8, 9


class Grid:
    """the blocks of every rank and the exchange between them"""

    def __init__(self, s, d, V, R, Cc, w=None, dtype=np.float32, device="cpu"):
        import torch
        from cugraph_b200 import _capi
        from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
        from cugraph_b200.pylibcugraph.utils import View
        self.torch, self.capi, self.View = torch, _capi, View
        self.L = _capi.lib()
        self.V, self.R, self.Cc, self.P = V, R, Cc, R * Cc
        self.device = device
        self.tt = torch.float32 if dtype == np.float32 else torch.float64
        self.es = 4 if dtype == np.float32 else 8
        owner = (np.arange(V, dtype=np.int64) * 2654435761 >> 7) % self.P
        order = np.argsort(owner, kind="stable")
        self.counts = np.bincount(owner, minlength=self.P)
        mp = self.mp = int(self.counts.max())
        lid = np.empty(V, dtype=np.int64)
        lid[order] = np.arange(V) - np.repeat(np.cumsum(self.counts) - self.counts, self.counts)
        self.own = [np.where(owner == p)[0][np.argsort(lid[owner == p])] for p in range(self.P)]
        r_of, c_of = owner // Cc, owner % Cc
        self.n_rows, self.n_cols = Cc * mp, R * mp
        self.handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
        self.err = C.c_void_p()
        self.blocks, self.keep, self.empty_blocks = {}, [], 0
        for r in range(R):
            for c in range(Cc):
                m = (r_of[d] == r) & (c_of[s] == c)
                self.empty_blocks += int(not m.any())
                rows = self.t((c_of[d[m]] * mp + lid[d[m]]).astype(np.int32))
                cols = self.t((r_of[s[m]] * mp + lid[s[m]]).astype(np.int32))
                ww = self.t(np.asarray(w[m], dtype=dtype)) if w is not None else None
                views = [View(rows), View(cols), View(ww)]
                blk = C.c_void_p()
                code = self.L.cugraph_b200_block_create(self.handle.ptr, self.n_rows, self.n_cols, views[0].ptr, views[1].ptr,
                                                        views[2].ptr, C.byref(blk), C.byref(self.err))
                _capi.check(code, self.err, "cugraph_b200_block_create")
                self.keep.append((rows, cols, ww, views))
                self.blocks[(r, c)] = blk.value
        self.span = int(self.L.cugraph_b200_block_span(self.blocks[(0, 0)]))
        self.x_elems = int(self.L.cugraph_b200_padded_elems(self.span, self.es))
        # one x and one y per block and orientation, kept across sweeps (the covered-rows state lives with the y)
        self.bufs = {}
        for key in self.blocks:
            for o in (0, 1):
                x = self.zeros(self.x_elems)
                y = self.zeros(self.span)
                self.bufs[key + (o,)] = (x, y, View(x), View(y))

    def t(self, a):
        return self.torch.as_tensor(np.ascontiguousarray(a)).to(self.device)

    def zeros(self, n, dtype=None):
        return self.torch.zeros(n, dtype=dtype or self.tt).to(self.device)

    def free(self):
        for blk in self.blocks.values():
            self.L.cugraph_b200_block_free(blk)
        for *_, views in self.keep:
            for v in views:
                v.free()
        for *_, vx, vy in self.bufs.values():
            vx.free()
            vy.free()

    def spmv(self, x_own, alpha, transposed=False, use_weights=True):
        """y_own[p] = alpha * (A x) (transposed: A^T x) of rank p's vertices, from the owners' x_own[p]"""
        torch, R, Cc, mp = self.torch, self.R, self.Cc, self.mp
        ys = {}
        for (r, c), blk in self.blocks.items():
            x, y, vx, vy = self.bufs[(r, c, int(transposed))]
            if transposed:   # all-gather in the row group: row slot c(v) * maxpart + lid
                gathered = torch.cat([x_own[r * Cc + cc] for cc in range(Cc)])
            else:            # all-gather in the column group: column slot r(u) * maxpart + lid
                gathered = torch.cat([x_own[rr * Cc + c] for rr in range(R)])
            x[:gathered.numel()].copy_(gathered)
            code = self.L.cugraph_b200_block_sweep(self.handle.ptr, blk, int(transposed), int(use_weights), vx.ptr, vy.ptr,
                                                   float(alpha), C.byref(self.err))
            self.capi.check(code, self.err, "cugraph_b200_block_sweep")
            ys[(r, c)] = y
        out = [None] * self.P
        if transposed:       # reduce-scatter in the column group
            for c in range(Cc):
                total = torch.stack([ys[(r, c)][:self.n_cols] for r in range(R)]).sum(0)
                for rr in range(R):
                    out[rr * Cc + c] = total[rr * mp:(rr + 1) * mp].clone()
        else:                # reduce-scatter in the row group
            for r in range(R):
                total = torch.stack([ys[(r, c)][:self.n_rows] for c in range(Cc)]).sum(0)
                for j in range(Cc):
                    out[r * Cc + j] = total[j * mp:(j + 1) * mp].clone()
        return out

    def step(self, name, *args):
        """one owner-step call; scalar tensors (scalars()) become double pointers, other tensors views (freed after the
        call); the rest is passed on"""
        conv, views = [], []
        for a in args:
            if getattr(a, "_scalars", False):
                conv.append(C.c_void_p(a.data_ptr()))
            elif isinstance(a, self.torch.Tensor):
                v = self.View(a)
                views.append(v)
                conv.append(v.ptr)
            else:
                conv.append(a)
        code = getattr(self.L, name)(self.handle.ptr, *conv, C.byref(self.err))
        for v in views:
            v.free()
        self.capi.check(code, self.err, name)

    def scalars(self, n):
        s = self.zeros(n, self.torch.float64)
        s._scalars = True
        return s

    def all_reduce(self, parts, op="sum"):
        """every rank's partial scalars -> the global value on every rank (in place)"""
        st = self.torch.stack(list(parts))
        tot = st.sum(0) if op == "sum" else st.max(0).values
        for p in parts:
            p.copy_(tot)
        return tot.cpu().numpy().astype(np.float64)

    def by_vertex(self, own_vals):
        out = np.zeros(self.V)
        for p in range(self.P):
            out[self.own[p]] = own_vals[p][:self.counts[p]].cpu().numpy()
        return out


def katz(grid, alpha, beta=1.0, epsilon=1e-6, max_iterations=100):
    """Returns (values by vertex id, iterations); the iteration of MGGraph.katz_centrality"""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    x = [grid.zeros(grid.mp) for _ in range(grid.P)]
    it = 0
    while True:
        y = grid.spmv(x, alpha)
        parts = [grid.scalars(2) for _ in range(grid.P)]
        for p in range(grid.P):
            grid.step("cugraph_b200_katz_step", y[p], x[p], int(grid.counts[p]), float(beta), parts[p])
        diff, sumsq = grid.all_reduce(parts)
        it += 1
        if T(diff) < T(epsilon):
            break
        if it >= max_iterations:
            raise RuntimeError("Katz Centrality failed to converge.")
    for p in range(grid.P):
        grid.step("cugraph_b200_vertex_scale", x[p], int(grid.counts[p]), 1.0 / float(np.sqrt(sumsq)))
    return grid.by_vertex(x), it


def eigenvector(grid, epsilon=1e-6, max_iterations=100):
    """Returns (values by vertex id, iterations); the iteration of MGGraph.eigenvector_centrality"""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    x = []
    for p in range(grid.P):
        xp = grid.zeros(grid.mp)
        xp[:grid.counts[p]] = 1.0 / grid.V
        x.append(xp)
    it = 0
    while True:
        y = grid.spmv(x, 1.0)
        sq = [grid.scalars(1) for _ in range(grid.P)]
        for p in range(grid.P):
            grid.step("cugraph_b200_eigenvector_add_step", y[p], x[p], int(grid.counts[p]), sq[p])
        grid.all_reduce(sq)
        parts = [grid.scalars(1) for _ in range(grid.P)]
        for p in range(grid.P):
            grid.step("cugraph_b200_eigenvector_scale_step", y[p], x[p], int(grid.counts[p]), sq[p], parts[p])
        diff, = grid.all_reduce(parts)
        it += 1
        if T(diff) < T(grid.V) * T(epsilon):
            break
        if it >= max_iterations:
            raise RuntimeError("Eigenvector Centrality failed to converge.")
    return grid.by_vertex(x), it


def hits(grid, epsilon=1e-5, max_iterations=100, initial_hubs=None, normalize=True):
    """Returns (hubs, authorities by vertex id, iterations, last difference); the iteration of MGGraph.hits.  initial_hubs:
    values by vertex id (already with the owners: MGGraph.hits moves them there with an all-to-all)"""
    T = np.float32 if grid.tt == grid.torch.float32 else np.float64
    P, mp = grid.P, grid.mp
    n = [int(c) for c in grid.counts]

    def l1(vecs):
        parts = [grid.scalars(1) for _ in range(P)]
        for p in range(P):
            grid.step("cugraph_b200_vertex_sum", vecs[p], n[p], 0, parts[p])
        norm, = grid.all_reduce(parts)
        assert T(norm) > 0
        for p in range(P):
            grid.step("cugraph_b200_vertex_scale", vecs[p], n[p], 1.0 / norm)

    prev = []
    for p in range(P):
        h = grid.zeros(mp)
        h[:n[p]] = 1.0 / grid.V if initial_hubs is None else grid.t(np.asarray(initial_hubs)[grid.own[p]].astype(T))
        prev.append(h)
    if initial_hubs is not None:
        l1(prev)
    it, diff = 0, 0.0
    while True:
        auth = grid.spmv(prev, 1.0, use_weights=False)
        curr = grid.spmv(auth, 1.0, transposed=True, use_weights=False)
        mx = [grid.scalars(2) for _ in range(P)]
        for p in range(P):
            grid.step("cugraph_b200_hits_max_step", curr[p], auth[p], n[p], mx[p])
        h_max, a_max = grid.all_reduce(mx, op="max")
        assert h_max > 0 and a_max > 0
        parts = [grid.scalars(1) for _ in range(P)]
        for p in range(P):
            grid.step("cugraph_b200_hits_scale_step", curr[p], auth[p], prev[p], n[p], mx[p], parts[p])
        d, = grid.all_reduce(parts)
        diff = float(T(d))
        prev = curr
        it += 1
        if T(diff) < T(grid.V) * T(epsilon):
            break
        if it >= max_iterations:
            raise RuntimeError("HITS failed to converge.")
    if normalize:
        l1(prev)
        l1(auth)
    return grid.by_vertex(prev), grid.by_vertex(auth), it, diff


# ---------------------------------------------------------------------------------------------------------------------
# single GPU, graphs, checks
# ---------------------------------------------------------------------------------------------------------------------
def single_gpu(algo, s, d, V, w=None, **kw):
    """cugraph_katz_centrality / _eigenvector_centrality / cugraph_hits on the same graph (every id 0..V-1 a vertex), by
    vertex id.  Katz and eigenvector: (values, None); HITS: (hubs, authorities)."""
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import by_vertex, make_graph
    wdt = np.float32 if w is None else w.dtype
    h, g = make_graph(s, d, weights=w, store_transposed=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=wdt)
    if algo == "katz":
        v, x = plc.katz_centrality(h, g, None, kw["alpha"], kw.get("beta", 1.0), kw["epsilon"], kw["max_iterations"], False)
        return by_vertex(v, x, V).astype(np.float64), None
    if algo == "eigenvector":
        v, x = plc.eigenvector_centrality(h, g, kw["epsilon"], kw["max_iterations"], False)
        return by_vertex(v, x, V).astype(np.float64), None
    v, hb, au = plc.hits(h, g, kw["epsilon"], kw["max_iterations"], None, None, True, False)
    return by_vertex(v, hb, V).astype(np.float64), by_vertex(v, au, V).astype(np.float64)


def katz_alpha(d, V):
    """api.katz_centrality's default on a directed graph: 1 / (1 + the largest in-degree)"""
    return 1.0 / (1.0 + float(np.bincount(d, minlength=V).max()))


def rmat_graph(scale, seed=900):
    """directed RMAT, ef 16"""
    from oracle.rmat import rmat_edgelist
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed + scale)
    return np.asarray(s, np.int32), np.asarray(d, np.int32), 1 << scale


def odd_graph(seed=7):
    """directed: a small RMAT, a chain, sources without in-edges, sinks without out-edges, a 2-cycle, duplicate edges and
    isolated ids, with the ids scattered"""
    from oracle.rmat import rmat_edgelist
    rs, rd = rmat_edgelist(6, 8 << 6, seed=seed)
    parts_s, parts_d = [np.asarray(rs, np.int64)], [np.asarray(rd, np.int64)]
    base = 1 << 6
    chain = np.arange(base, base + 20)
    parts_s += [chain[:-1], np.full(10, chain[0])]                 # the chain and a fan out of its head
    parts_d += [chain[1:], np.arange(base + 20, base + 30)]        # the fan's leaves are sinks
    base += 30
    parts_s += [np.arange(base, base + 8), np.array([base + 8, base + 9, base + 8])]   # 8 sources into the RMAT part
    parts_d += [np.arange(8), np.array([base + 9, base + 8, base + 9])]                # a 2-cycle with a duplicate edge
    base += 10
    V = base + 6                                                  # the last six ids are isolated
    s, d = np.concatenate(parts_s), np.concatenate(parts_d)
    perm = np.random.default_rng(seed).permutation(V)
    return perm[s].astype(np.int32), perm[d].astype(np.int32), V


def tiny_graph():
    """five edges over 12 vertices: on a 4x2 grid most blocks have no edges"""
    s = np.array([0, 1, 5, 9, 2], np.int32)
    d = np.array([1, 5, 9, 2, 0], np.int32)
    return s, d, 12
