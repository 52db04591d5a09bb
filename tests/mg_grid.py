"""All P = R x C ranks of a 2D edge partition in ONE process: the simulated grid under the one-process multi-GPU tests
(tests/test_emu_mg_cpu.py, tests/mg_sssp_sim.py, tests/mg_wcc_sim.py, tests/mg_centrality_sim.py).  Every rank's block goes
through the real block entry points; the all-gathers, reduce-scatters and all-reduces between them are tensor ops on one
device, in the groups MGGraph uses.  Torch CPU tensors with the emulated library (tests/emu_py.py) or CUDA tensors with the
real one.

The partition: every id 0..V-1 is a vertex; vertex v belongs to rank owner(v) = (v * 2654435761 >> 7) % P at grid position
(r(v), c(v)) = (owner // C, owner % C), with local ids in id order.  Edge (u -> v) lives on rank (r(v), c(u)), at row slot
c(v) * maxpart + lid(v) and column slot r(u) * maxpart + lid(u); rank p's code for its vertex of local id l is p * maxpart + l.
"""
import ctypes as C

import numpy as np


class Grid:
    """the blocks of every rank and the exchange between them"""

    def __init__(self, s, d, V, R, Cc, w=None, dtype=None, device="cpu"):
        import torch
        from cugraph_b200 import _capi
        from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
        from cugraph_b200.pylibcugraph.utils import View
        self.torch, self.capi, self.View = torch, _capi, View
        self.L = _capi.lib()
        self.V, self.R, self.Cc, self.P = V, R, Cc, R * Cc
        self.device = device
        dtype = np.dtype(dtype or (w.dtype if w is not None else np.float32))
        self.tt = torch.float32 if dtype == np.float32 else torch.float64
        # the partition
        owner = (np.arange(V, dtype=np.int64) * 2654435761 >> 7) % self.P
        order = np.argsort(owner, kind="stable")
        self.counts = np.bincount(owner, minlength=self.P)
        mp = self.mp = int(self.counts.max())
        lid = np.empty(V, dtype=np.int64)
        lid[order] = np.arange(V) - np.repeat(np.cumsum(self.counts) - self.counts, self.counts)
        self.owner, self.lid = owner, lid
        self.own = [np.where(owner == p)[0][np.argsort(lid[owner == p])] for p in range(self.P)]   # vertex ids by local id
        self.code_vertex = np.full(self.P * mp, -1, dtype=np.int64)                                 # code -> vertex id
        for p in range(self.P):
            self.code_vertex[p * mp:p * mp + self.counts[p]] = self.own[p]
        r_of, c_of = owner // Cc, owner % Cc
        self.n_rows, self.n_cols = Cc * mp, R * mp
        # the blocks
        self.handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
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
                self.call("cugraph_b200_block_create", self.n_rows, self.n_cols, views[0].ptr, views[1].ptr, views[2].ptr,
                          C.byref(blk))
                self.keep.append((rows, cols, ww, views))
                self.blocks[(r, c)] = blk.value
        self.span = int(self.L.cugraph_b200_block_span(self.blocks[(0, 0)]))
        self.x_elems = int(self.L.cugraph_b200_padded_elems(self.span, dtype.itemsize))
        # one x and one y per block and orientation, kept across sweeps (the covered-rows state lives with the y)
        self.bufs = {key + (o,): (self.zeros(self.x_elems), self.zeros(self.span)) for key in self.blocks for o in (0, 1)}

    def t(self, a):
        return self.torch.as_tensor(np.ascontiguousarray(a)).to(self.device)

    def zeros(self, n, dtype=None):
        return self.torch.zeros(n, dtype=dtype or self.tt).to(self.device)

    def scalars(self, n):
        """n device doubles that call() passes as a double pointer"""
        s = self.zeros(n, self.torch.float64)
        s._scalars = True
        return s

    def free(self):
        for blk in self.blocks.values():
            self.L.cugraph_b200_block_free(blk)
        for *_, views in self.keep:
            for v in views:
                v.free()

    def call(self, name, *args):
        """one entry-point call on the grid's handle: scalar tensors (scalars()) become double pointers, other tensors views
        (freed after the call); the rest is passed on"""
        conv, views = [], []
        for a in args:
            if getattr(a, "_scalars", False):
                conv.append(C.c_void_p(a.data_ptr()))
            elif isinstance(a, self.torch.Tensor):
                views.append(self.View(a))
                conv.append(views[-1].ptr)
            else:
                conv.append(a)
        err = C.c_void_p()
        code = getattr(self.L, name)(self.handle.ptr, *conv, C.byref(err))
        for v in views:
            v.free()
        self.capi.check(code, err, name)

    # ---- collectives
    def gather(self, own, r, c, rows=False):
        """the owners' `own` over block (r, c)'s column slots (the column group's all-gather) or, rows=True, over its row
        slots (the row group's all-gather)"""
        if rows:
            return self.torch.cat([own[r * self.Cc + cc] for cc in range(self.Cc)])
        return self.torch.cat([own[rr * self.Cc + c] for rr in range(self.R)])

    def reduce_scatter(self, parts, op="sum", rows=True):
        """every block's parts[(r, c)] over its row slots reduced inside the row group (rows=False: over its column slots,
        inside the column group) -> each rank's maxpart slice, by rank"""
        torch, mp = self.torch, self.mp
        out = [None] * self.P
        groups = [[(r, c) for c in range(self.Cc)] for r in range(self.R)] if rows else \
                 [[(r, c) for r in range(self.R)] for c in range(self.Cc)]
        n = self.n_rows if rows else self.n_cols
        for keys in groups:
            st = torch.stack([parts[k][:n] for k in keys])
            total = st.sum(0) if op == "sum" else st.min(0).values if op == "min" else st.max(0).values
            for j, (r, c) in enumerate(keys):
                out[r * self.Cc + j if rows else j * self.Cc + c] = total[j * mp:(j + 1) * mp].clone()
        return out

    def all_reduce(self, parts, op="sum"):
        """every rank's partial scalars -> the global value on every rank (in place)"""
        st = self.torch.stack(list(parts))
        tot = st.sum(0) if op == "sum" else st.max(0).values
        for p in parts:
            p.copy_(tot)
        return tot.cpu().numpy().astype(np.float64)

    def spmv(self, x_own, alpha, transposed=False, use_weights=True):
        """y_own[p] = alpha * (A x) (transposed: A^T x) of rank p's vertices, from the owners' x_own[p]: a pull sweep gathers
        x in the column group and reduces y in the row group, a transposed sweep the other way round"""
        ys = {}
        for (r, c), blk in self.blocks.items():
            x, y = self.bufs[(r, c, int(transposed))]
            g = self.gather(x_own, r, c, rows=transposed)
            x[:g.numel()].copy_(g)
            self.call("cugraph_b200_block_sweep", blk, int(transposed), int(use_weights), x, y, float(alpha))
            ys[(r, c)] = y
        return self.reduce_scatter(ys, rows=not transposed)

    # ---- results
    def by_vertex(self, own_vals, dtype=np.float64):
        """the owners' values (each rank's first counts[p] entries) indexed by vertex id"""
        out = np.zeros(self.V, dtype=dtype)
        for p in range(self.P):
            out[self.own[p]] = own_vals[p][:self.counts[p]].cpu().numpy()
        return out

    def vertex_of(self, codes):
        """vertex codes (rank * maxpart + local id) -> vertex ids; negative codes stay -1"""
        codes = np.asarray(codes, dtype=np.int64)
        return np.where(codes >= 0, self.code_vertex[np.maximum(codes, 0)], -1)
