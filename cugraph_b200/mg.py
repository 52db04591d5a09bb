"""Multi-GPU PageRank, BFS, SSSP, weakly and strongly connected components, Katz, eigenvector centrality and HITS: 2D edge partition over one process per GPU (torch.distributed, NCCL on NVLink 5).

What the reference does (SURVEY.md §8e): P = R x C GPUs, vertex -> GPU by hash
(cpp/include/cugraph/utilities/graph_partition_utils.cuh:30-43, 101-128), every GPU holds the edge
block (row block of destinations) x (column block of sources); per PageRank iteration the scaled
ranks are all-gathered inside the column group (update_edge_src_property, grouped ncclBroadcast,
update_edge_src_dst_property.cuh:550-579), the local pull sweep runs, and the partial sums are reduced
to their owners inside the row group (grouped ncclReduce, per_v_transform_reduce_e.cuh:3389-3407).

Here: the same partition, but the exchange is ONE all_gather_into_tensor + ONE reduce_scatter_tensor
per iteration on equal-sized (padded) vertex partitions, the dangling / convergence scalars travel in
one 2-element all_reduce and never touch the host unless epsilon > 0, and the local sweep is the
same column-blocked shared-memory kernel as on one GPU (C-ABI: cugraph_b200_block_*).

BFS moves byte flags per level (one max-reduce-scatter of candidate predecessors), from one source or a set of sources
given by every rank (multi_source_bfs: one BFS per source, 64-bit words per vertex for a batch of 64, see
MGGraph.multi_source_bfs); extract_paths walks the BFS predecessors one path position per round, each an all-to-all-v of local
ids to their owners and one of (external id, predecessor code) answers back (see MGGraph.extract_paths); SSSP runs
Δ-windows of rounds, each an all-gather of the frontier's distances, the block's push relaxation on the device and one
min-reduce-scatter of INT64 (distance, predecessor) keys (see MGGraph.sssp); WCC propagates the smallest vertex code per round, with one
min-reduce-scatter of INT64 labels (see MGGraph.weakly_connected_components); SCC runs single GPU's Multistep phases as
rounds of block pushes in both directions, forward through the block's column-major copy and backward through its own rows
(see _SccRun); Katz, eigenvector centrality and HITS iterate
the block sweep like PageRank, HITS also in the transposed orientation, with owner-step kernels between the collectives
(see MGGraph.katz_centrality).

`partition_edges` (pure torch, device agnostic: exercised on CPU with the gloo backend in
tests/test_mg_partition_cpu.py) builds the blocks; `MGGraph` and the module-level algorithm functions need CUDA.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import math
import os
from dataclasses import dataclass

import numpy as np
import torch
import torch.distributed as dist


# ----------------------------------------------------------------------------------------------
# process grid (reference: cpp/tests/utilities/mg_utilities.cpp:49-53, partition_manager.hpp:106-114)
# ----------------------------------------------------------------------------------------------
def grid_shape(world: int):
    """(R, C) of the P = R x C process grid: R = size of the all-gather (column) group, C = size of the reduce (row) group.
    The two factors are the reference's (largest divisor <= sqrt(P) and its cofactor, mg_utilities.cpp:49-53); the LARGER one
    is R here: 2 -> 2x1, 4 -> 2x2, 8 -> 4x2.  A GPU's block has C * maxpart destination rows and R * maxpart source columns.
    The number of pieces (= accumulations) of a block does not depend on the orientation (numpy count on RMAT, scale 20 per
    GPU: 1x2 5.12 M pieces / 2x1 5.20 M; 2x4 6.88 M / 4x2 6.98 M) but its rows do: with R >= C the accumulator array and
    the finish pass are half (N = 2, 8) the size — 70 MB instead of 141 MB of accumulators at RMAT-25 on 2 GPUs, i.e. inside
    the L2 again.  CUGRAPH_B200_MG_GRID=wide restores the reference's orientation (R <= C)."""
    r = int(math.isqrt(world))
    while world % r:
        r -= 1
    small, large = r, world // r
    if os.environ.get("CUGRAPH_B200_MG_GRID", "tall") == "wide":
        return small, large
    return large, small


def vertex_owner(ext: torch.Tensor, world: int) -> torch.Tensor:
    """Balanced vertex -> GPU map (the role of murmurhash3_32(ext) % P in the reference)."""
    x = ext.to(torch.int64)
    x = (x ^ (x >> 30)) * -4658895280553007687   # 0xbf58476d1ce4e5b9 as int64
    x = (x ^ (x >> 27)) * -7723592293110705685   # 0x94d049bb133111eb as int64
    x = x ^ (x >> 31)
    return (x & 0x7FFFFFFFFFFFFFFF) % world


@dataclass
class Groups:
    world: int
    rank: int
    R: int
    C: int
    r: int
    c: int
    row_group: object   # ranks (r, *)  : reduce-scatter of partial y
    col_group: object   # ranks (*, c)  : all-gather of x


def make_groups() -> Groups:
    world, rank = dist.get_world_size(), dist.get_rank()
    R, Cc = grid_shape(world)
    r, c = rank // Cc, rank % Cc
    row_group = col_group = None
    for rr in range(R):
        g = dist.new_group([rr * Cc + cc for cc in range(Cc)])
        if rr == r:
            row_group = g
    for cc in range(Cc):
        g = dist.new_group([rr * Cc + cc for rr in range(R)])
        if cc == c:
            col_group = g
    return Groups(world, rank, R, Cc, r, c, row_group, col_group)


# ----------------------------------------------------------------------------------------------
# collectives that also run on gloo (CPU tests)
# ----------------------------------------------------------------------------------------------
def _is_nccl(group=None):
    return dist.get_backend(group) == "nccl"


def exchange(tensors, dest: torch.Tensor, world: int):
    """all-to-all-v: element i of every tensor goes to rank dest[i]. Returns received tensors."""
    order = torch.argsort(dest, stable=True)
    send_counts = torch.bincount(dest, minlength=world).to(torch.int64)
    recv_counts = torch.empty_like(send_counts)
    dist.all_to_all_single(recv_counts, send_counts)
    sc, rc = send_counts.tolist(), recv_counts.tolist()
    out = []
    for t in tensors:
        ts = t[order].contiguous()
        tr = torch.empty(sum(rc), dtype=t.dtype, device=t.device)
        dist.all_to_all_single(tr, ts, output_split_sizes=rc, input_split_sizes=sc)
        out.append(tr)
    return out, order, sc, rc


def all_gather_into(out: torch.Tensor, inp: torch.Tensor, group):
    """out = every member's inp, in group-rank order.  A one-member group copies: no collective call."""
    if dist.get_world_size(group) == 1:
        out.copy_(inp)
    elif _is_nccl(group):
        dist.all_gather_into_tensor(out, inp, group=group)
    else:
        n = dist.get_world_size(group)
        parts = [torch.empty_like(inp) for _ in range(n)]
        dist.all_gather(parts, inp, group=group)
        out.copy_(torch.cat(parts))


def reduce_scatter_into(out: torch.Tensor, inp: torch.Tensor, group, op=None):
    """out = this member's slice of the members' inp reduced with op (default SUM).  A one-member group copies: no
    collective call."""
    op = op or dist.ReduceOp.SUM
    if dist.get_world_size(group) == 1:
        out.copy_(inp)
    elif _is_nccl(group):
        dist.reduce_scatter_tensor(out, inp, op=op, group=group)
    else:
        tmp = inp.clone()
        dist.all_reduce(tmp, op=op, group=group)
        k = dist.get_rank(group)
        out.copy_(tmp[k * out.numel():(k + 1) * out.numel()])


def _unique_big(tensors, chunk=1 << 29):
    """sorted unique of the concatenation, in pieces (torch.unique is limited to < 2^31 elements)."""
    parts = []
    for t in tensors:
        for i in range(0, max(t.numel(), 1), chunk):
            parts.append(torch.unique(t[i:i + chunk]))
    while len(parts) > 1:
        parts = [torch.unique(torch.cat(parts[i:i + 2])) for i in range(0, len(parts), 2)]
    return parts[0]


# ----------------------------------------------------------------------------------------------
# 2D partition
# ----------------------------------------------------------------------------------------------
# the most shuffled edges per GPU that cugraph_b200_block_stage_edges takes (single-GPU staging's bounds): 2n < 2^31 with
# symmetrize, n < 2^32 with weights
STAGE_MAX_SYMMETRIZED = (1 << 30) - 1
STAGE_MAX_WEIGHTED = (1 << 32) - 1


@dataclass
class Partition:
    groups: Groups
    rows: torch.Tensor        # int32, local destination slot of every local edge: c_v * maxpart + lid
    cols: torch.Tensor        # int32, local source slot: r_u * maxpart + lid (partition-major: the all-gather output order)
    weights: object           # tensor or None
    vertices: torch.Tensor    # external ids of the vertices this rank owns, in local-id order
    n_local: int
    maxpart: int
    n_global: int
    reversed: object = None   # uint8 per local edge with symmetrize: 1 = the reversed copy of an edge v -> u, else None


def partition_edges(src: torch.Tensor, dst: torch.Tensor, weights=None, groups: Groups | None = None, *, vertices=None,
                    drop_self_loops=False, drop_multi_edges=False, symmetrize=False) -> Partition:
    """Shuffle this rank's share of the edge list into the 2D partition and renumber.
    Edge (u -> v) is stored on GPU (r(owner(v)), c(owner(u)))  (graph_partition_utils.cuh:101-128).
    vertices: external ids (the edge ids' dtype) that are vertices also without an edge, sent to their owners with the
    referenced ids; drop_self_loops: edges u -> u are dropped first; symmetrize: a reversed copy v -> u of every other edge
    travels with it, flagged in Partition.reversed (MGGraph stages the block from them).  drop_multi_edges changes nothing
    here; with it or symmetrize, the size bounds of cugraph_b200_block_stage_edges are checked on the shuffled edges.  Every
    rank raises the same error, after the one MAX all-reduce that also gives maxpart: TypeError for a `vertices` dtype that
    differs from the edge ids' on some rank, ValueError for a rank with too many shuffled edges to stage."""
    g = groups or make_groups()
    P, Cc = g.world, g.C
    bad_vertices = 0
    if vertices is not None:
        vertices = torch.as_tensor(vertices)
        if vertices.dtype != src.dtype:
            bad_vertices, vertices = 1, None     # sent as none; every rank raises after the all-reduce below
        else:
            vertices = torch.unique(vertices.to(src.device).reshape(-1))
    if drop_self_loops:
        keep = src != dst
        src, dst = src[keep], dst[keep]
        weights = weights[keep] if weights is not None else None
    rev = None
    if symmetrize:
        other = src != dst
        n_rev = int(other.sum().item())
        src, dst = torch.cat([src, dst[other]]), torch.cat([dst, src[other]])
        weights = torch.cat([weights, weights[other]]) if weights is not None else None
        rev = torch.cat([torch.zeros(src.numel() - n_rev, dtype=torch.uint8, device=src.device),
                         torch.ones(n_rev, dtype=torch.uint8, device=src.device)])
    so, do = vertex_owner(src, P), vertex_owner(dst, P)
    target = (do // Cc) * Cc + (so % Cc)
    payload = [src, dst] + ([weights] if weights is not None else []) + ([rev] if rev is not None else [])
    recv, _, _, _ = exchange(payload, target, P)
    src_e, dst_e = recv[0], recv[1]
    w_e = recv[2] if weights is not None else None
    rev_e = recv[-1] if rev is not None else None
    # vertices referenced here -> their owners, together with how often each is a SOURCE here; the owner
    # numbers its vertices by descending global out-degree so that hot sources get the lowest local ids
    # (the column-blocked sweep keeps the lowest column ids in shared memory) — the role of the
    # reference's per-GPU degree-descending renumbering (renumber_edgelist_impl.cuh:732-738)
    u = _unique_big([src_e, dst_e])
    ks = torch.searchsorted(u, src_e)
    cnt = torch.bincount(ks, minlength=u.numel()).to(torch.int64)
    ids, ids_cnt = u, cnt
    if vertices is not None:   # listed vertices travel with the referenced ids, as sources of no edge
        ids = torch.cat([u, vertices])
        ids_cnt = torch.cat([cnt, torch.zeros(vertices.numel(), dtype=torch.int64, device=cnt.device)])
    ou = vertex_owner(ids, P)
    (recv_ids, recv_cnt), order, sc, rc = exchange([ids, ids_cnt], ou, P)
    mine, inv = torch.unique(recv_ids, return_inverse=True)   # sorted external ids owned by this rank
    n_local = int(mine.numel())
    deg = torch.zeros(n_local, dtype=torch.int64, device=src.device).index_add_(0, inv, recv_cnt)
    by_deg = torch.argsort(-deg, stable=True)                  # by_deg[l] = index into `mine` of local id l
    lid_of_mine = torch.empty_like(by_deg)
    lid_of_mine[by_deg] = torch.arange(n_local, device=src.device)
    pos = lid_of_mine[inv]                                     # local id of every requested vertex
    mine = mine[by_deg]                                        # external ids in local-id order
    back = torch.empty(sum(sc), dtype=pos.dtype, device=pos.device)
    dist.all_to_all_single(back, pos.contiguous(), output_split_sizes=sc, input_split_sizes=rc)
    lid = torch.empty_like(back)
    lid[order] = back                                   # lid[k] = local id (at its owner) of u[k]
    t = torch.tensor([n_local, n_local], dtype=torch.int64, device=src.device)
    n_e = src_e.numel()
    too_many = int((symmetrize and n_e > STAGE_MAX_SYMMETRIZED) or
                   ((symmetrize or drop_multi_edges) and weights is not None and n_e > STAGE_MAX_WEIGHTED))
    mx = torch.tensor([n_local, bad_vertices, too_many], dtype=torch.int64, device=src.device)   # input errors ride along
    dist.all_reduce(mx, op=dist.ReduceOp.MAX)
    if int(mx[1].item()):
        raise TypeError("MGGraph: vertices must have the dtype of the edge ids on every rank")
    if int(mx[2].item()):
        raise ValueError("MGGraph: too many edges on one GPU to stage (symmetrize needs 2n < 2^31, weighted multi-edge "
                         "removal n < 2^32 shuffled edges per GPU)")
    tot = t[1:].clone()
    dist.all_reduce(tot, op=dist.ReduceOp.SUM)
    maxpart = max(int(mx[0].item()), 1)
    kd = torch.searchsorted(u, dst_e)
    rows = ((ou[kd] % Cc) * maxpart + lid[kd]).to(torch.int32)
    # columns are partition-major (slot = r_u * maxpart + lid): exactly the layout all_gather_into_tensor produces, so the
    # gathered x is consumed in place (an interleaved order put all hot sources into the first column block but cost a
    # strided 4 * n_cols-byte transpose copy per iteration; every partition's hot sources still lead ITS column range)
    cols = ((ou[ks] // Cc) * maxpart + lid[ks]).to(torch.int32)
    return Partition(g, rows, cols, w_e, mine, n_local, maxpart, int(tot.item()), rev_e)


# ----------------------------------------------------------------------------------------------
# CUDA side
# ----------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _views(*tensors):
    """C array views of the tensors (None gives a NULL view), freed when the block exits, also when it raises"""
    from cugraph_b200.pylibcugraph.utils import View
    vs = []
    try:
        for t in tensors:
            vs.append(View(t))
        yield vs
    finally:
        for v in vs:
            v.free()


def _global_count(mask):
    """the number of set entries of `mask` over all ranks, as a host int (one all-reduce)"""
    n = mask.sum().to(torch.int64).reshape(1)
    dist.all_reduce(n)
    return int(n.item())


class MGGraph:
    """This rank's edge block of a 2D-partitioned graph (pull orientation: rows = destinations).

    src, dst (and weights) are this rank's share of the edge list, in external ids.  The keyword options are those of the
    single-GPU constructor (cugraph_graph_create_sg), applied in the reference's order, and must be the same on every rank
    (not checked: with drop_self_loops or symmetrize differing between ranks the shuffle's collectives do not match):
      vertices: external ids, in the edge ids' dtype, that are vertices of the graph also without an edge (any rank may pass
        any ids, or None; duplicates are merged).  The vertices are these and the endpoints of the edges left after
        self-loop removal.
      drop_self_loops: edges u -> u are dropped.
      drop_multi_edges: one edge per (u, v) is kept, the one of MINIMUM weight, whatever order the edges arrive in.  Single
        GPU keeps the minimum only for a graph declared symmetric and otherwise the first copy in input order.
      symmetrize: single GPU's pairing rule: the edges between u and v are grouped, the i-th lightest u -> v edge paired with
        the i-th lightest v -> u edge becomes one undirected edge of the averaged weight (W)((a + b) / 2), unpaired edges keep
        their weight; every undirected edge is stored in both directions, a self-loop once.
    Errors raise on every rank: TypeError for a `vertices` dtype other than the edge ids' on any rank, ValueError for a rank
    with more shuffled edges than staging takes (see partition_edges), and a CugraphError when staging fails on some rank
    (that rank's own error, CugraphRuntimeError on the others; with drop_multi_edges or symmetrize only: one all-reduce of
    the outcome).  With every option at its default the construction is the plain shuffle of the edges as given."""

    def __init__(self, src, dst, weights=None, groups: Groups | None = None, dtype=torch.float32, *, vertices=None,
                 drop_self_loops=False, drop_multi_edges=False, symmetrize=False):
        from cugraph_b200 import _capi
        from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
        assert src.is_cuda or _capi.emulated(), "MGGraph needs CUDA tensors"
        self.lib = _capi.lib()
        self._capi = _capi
        self.dtype = dtype if weights is None else weights.dtype
        self.symmetrize = symmetrize   # strongly_connected_components rejects symmetric graphs, as on one GPU
        self.part = partition_edges(src, dst, weights, groups, vertices=vertices, drop_self_loops=drop_self_loops,
                                    drop_multi_edges=drop_multi_edges, symmetrize=symmetrize)
        p = self.part
        g = p.groups
        self.handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
        self.n_rows, self.n_cols = g.C * p.maxpart, g.R * p.maxpart
        if drop_multi_edges or symmetrize:
            self._stage_edges(drop_multi_edges, symmetrize)
        es = 4 if self.dtype == torch.float32 else 8
        blk = C.c_void_p()
        with _views(p.rows, p.cols, p.weights) as (rv, cv, wv):
            self._call("cugraph_b200_block_create", self.n_rows, self.n_cols, rv.ptr, cv.ptr, wv.ptr, C.byref(blk))
        self.block = blk.value
        self.span = int(self.lib.cugraph_b200_block_span(self.block))
        self.x_elems = int(self.lib.cugraph_b200_padded_elems(self.span, es))
        # out-weight sums of the owned vertices: partial per column slot, reduce-scattered in the column group
        ones = p.weights.to(torch.float64) if p.weights is not None else torch.ones(p.cols.numel(), dtype=torch.float64, device=src.device)
        partial = torch.zeros(self.n_cols, dtype=torch.float64, device=src.device)
        partial.index_add_(0, p.cols.long(), ones)                          # partition-major already
        ow = torch.empty(p.maxpart, dtype=torch.float64, device=src.device)
        reduce_scatter_into(ow, partial, g.col_group)
        self.out_w = ow.to(self.dtype)
        self.num_edges_local = int(p.rows.numel())
        self.weighted = p.weights is not None
        self._w_sum_local = float(ones.sum().item()) if self.weighted else 0.0   # SSSP's initial window width
        self._sssp_avg = None                                                       # (average weight, average degree)
        self._id_order = None                                  # (local ids by external id, sorted external ids)
        self.last_bfs_stats = None
        self.last_ms_bfs_stats = None
        self.last_sssp_stats = None
        self.last_wcc_stats = None
        self.last_scc_stats = None
        self.last_paths_stats = None
        self.last_katz_stats = self.last_eigenvector_stats = self.last_hits_stats = None
        self._degrees = None                                   # (in, out) of the owned slice, made by the first degrees()
        self.device = src.device
        p.rows = p.cols = p.weights = None  # the block owns its own copy
        torch.cuda.synchronize()

    def _stage_edges(self, drop_multi_edges, symmetrize):
        """multi-edge removal and symmetrization of this rank's shuffled edges, on the device (cugraph_b200_block_stage_edges,
        in place): every copy of u -> v, and with symmetrize every reversed copy of v -> u, is on this rank already"""
        p = self.part
        n_out = C.c_size_t()
        failure = None
        try:
            with _views(p.rows, p.cols, p.reversed, p.weights) as (rv, cv, fv, wv):
                self._call("cugraph_b200_block_stage_edges", self.n_rows, self.n_cols, rv.ptr, cv.ptr, fv.ptr, wv.ptr,
                           1 if drop_multi_edges else 0, 1 if symmetrize else 0, C.byref(n_out))
        except self._capi.CugraphError as e:   # e.g. out of memory on this rank alone: the others must not go on
            failure = e
        failed = torch.tensor([0 if failure is None else 1], dtype=torch.int64, device=p.rows.device)
        dist.all_reduce(failed, op=dist.ReduceOp.MAX)
        if failure is not None:
            raise failure
        if int(failed.item()):
            raise self._capi.CugraphRuntimeError(self._capi.UNKNOWN_ERROR, "staging the edges failed on another rank",
                                                 "MGGraph")
        m = n_out.value
        p.rows, p.cols = p.rows[:m], p.cols[:m]
        p.weights = p.weights[:m] if p.weights is not None else None
        p.reversed = None

    def degrees(self):
        """(vertices, in_degrees, out_degrees) of the vertices this rank owns: edge counts of the staged graph, in the
        vertices' dtype (single-GPU cugraph_degrees').  The first call counts the block's rows and columns
        (cugraph_b200_block_degrees) and reduce-scatters them in the row and the column group; later calls reuse the result."""
        p, g = self.part, self.part.groups
        if self._degrees is None:
            rows = torch.empty(self.n_rows, dtype=torch.int64, device=self.device)
            cols = torch.empty(self.n_cols, dtype=torch.int64, device=self.device)
            with _views(rows, cols) as (vr, vc):
                self._call("cugraph_b200_block_degrees", self.block, vr.ptr, vc.ptr)
            deg_in = torch.empty(p.maxpart, dtype=torch.int64, device=self.device)
            deg_out = torch.empty(p.maxpart, dtype=torch.int64, device=self.device)
            reduce_scatter_into(deg_in, rows, g.row_group)
            reduce_scatter_into(deg_out, cols, g.col_group)                   # partition-major, as out_w
            dt = p.vertices.dtype
            self._degrees = (deg_in[:p.n_local].to(dt), deg_out[:p.n_local].to(dt))
        return p.vertices, self._degrees[0].clone(), self._degrees[1].clone()

    def __del__(self):
        try:
            if getattr(self, "block", None):
                self.lib.cugraph_b200_block_free(self.block)
                self.block = None
        except Exception:
            pass

    # one PageRank iteration = all-gather(x) -> block sweep -> reduce-scatter(y) -> vertex step -> all-reduce(2 scalars)
    def pagerank(self, alpha=0.85, epsilon=1e-5, max_iterations=100, *, personalization=None, initial_guess=None,
                 precomputed_out_weights=None, fail_on_nonconvergence=False):
        """PageRank of the vertices this rank owns: returns (vertices, values, iterations, converged).

        personalization, initial_guess and precomputed_out_weights are each a pair (external vertex ids, values), or None.
        Any rank may pass pairs for any vertices; an argument counts as given when some rank passes it.  As on one GPU:
        personalization teleports only to its vertices, in proportion to their values (cugraph_personalized_pagerank);
        initial_guess is the starting vector as given, without normalisation, 0 for vertices it does not name;
        precomputed_out_weights replace the out-weight sums, 0 (dangling) for vertices it does not name.  Every rank raises
        the same error for an invalid argument (see _pagerank_inputs).  fail_on_nonconvergence: FailedToConvergeError on
        every rank when max_iterations pass without convergence."""
        p, g = self.part, self.part.groups
        dev, dt, mp = self.out_w.device, self.dtype, p.maxpart
        given = torch.tensor([a is not None for a in (personalization, initial_guess, precomputed_out_weights)],
                             dtype=torch.int64, device=dev)
        dist.all_reduce(given, op=dist.ReduceOp.MAX)   # a pair from any rank: every rank takes part in its exchange
        pers, pers_sum, guess, out_w = None, 0.0, None, self.out_w
        flags = given.tolist()
        if any(flags):
            pers, pers_sum, guess, ow = self._pagerank_inputs((personalization, initial_guess, precomputed_out_weights), flags)
            out_w = self.out_w if ow is None else ow
        if guess is not None:
            pr = guess
        else:
            pr = torch.zeros(mp, dtype=dt, device=dev)
            pr[:p.n_local] = 1.0 / p.n_global
        x_local = torch.zeros(mp, dtype=dt, device=dev)
        xg = torch.zeros(self.x_elems, dtype=dt, device=dev)
        ypart = torch.zeros(self.span, dtype=dt, device=dev)
        yred = torch.zeros(mp, dtype=dt, device=dev)
        tot = torch.zeros(2, dtype=torch.float64, device=dev)
        part = torch.zeros(2, dtype=torch.float64, device=dev)
        pending = [None]

        with _views(pr, x_local, xg, ypart, yred, out_w, pers) as (vpr, vx, vxg, vyp, vyr, vow, vpers):
            def vertex_step(first):
                # the totals of the previous step are needed now: their all-reduce ran under the sweep in between
                if pending[0] is not None:
                    pending[0].wait()
                    pending[0] = None
                part.zero_()
                if pers is None:
                    self._call("cugraph_b200_pagerank_vertex_step", vyr.ptr, vpr.ptr, vow.ptr, vx.ptr, p.n_local,
                               float(alpha), float(p.n_global), 1 if first else 0, C.c_void_p(tot.data_ptr()),
                               C.c_void_p(part.data_ptr()))
                else:
                    self._call("cugraph_b200_pagerank_personalized_vertex_step", vyr.ptr, vpr.ptr, vow.ptr, vx.ptr,
                               vpers.ptr, p.n_local, float(alpha), pers_sum, 1 if first else 0, C.c_void_p(tot.data_ptr()),
                               C.c_void_p(part.data_ptr()))
                pending[0] = dist.all_reduce(part, async_op=True)

            vertex_step(True)
            tot, part = part, tot
            iters = 0
            xcols = xg[:self.n_cols]
            for _ in range(int(max_iterations)):
                all_gather_into(xcols, x_local, g.col_group)            # partition-major = the block's column order
                self._call("cugraph_b200_block_pull_sweep", self.block, vxg.ptr, vyp.ptr, float(alpha))
                reduce_scatter_into(yred, ypart[:self.n_rows], g.row_group)
                vertex_step(False)
                tot, part = part, tot
                iters += 1
                if epsilon > 0.0:   # host sync only when a tolerance is requested
                    pending[0].wait()
                    pending[0] = None
                    if float(tot[0].item()) < epsilon:
                        break
            if pending[0] is not None:
                pending[0].wait()
        converged = iters < max_iterations
        if fail_on_nonconvergence and not converged:   # every rank ran the same iterations: every rank raises
            from cugraph_b200.pylibcugraph.exceptions import FailedToConvergeError
            raise FailedToConvergeError(f"MGGraph.pagerank: PageRank failed to converge in {iters} iterations.")
        return p.vertices, pr[:p.n_local].clone(), iters, converged

    def _pagerank_inputs(self, args, given):
        """MGGraph.pagerank's (personalization, initial guess, precomputed out-weights) pairs -> (pers, pers_sum, guess,
        out_w) over this rank's owned slice (None where the argument is not given).  `given` says which arguments some rank
        passed.  Each given argument takes one all-to-all-v to the owners; one all-reduce then gathers every rank's error
        counts and the personalization sum, and every rank raises the first failing check in this order:
          personalization: ids and values differ in size on some rank; no pair on any rank; an id that is not a vertex; a
            negative value; an id given twice; a sum that is not positive  (the single-GPU messages and exception types,
            the reference's multi-GPU checks of pagerank_impl.cuh for the negative values and duplicates)
          initial guess, then precomputed out-weights: sizes differ; an id that is not a vertex."""
        from cugraph_b200 import _capi as capi
        dev, dt, mp = self.device, self.dtype, self.part.maxpart
        got, counts = [], []
        for a, f in zip(args, given):
            if f:
                lid, val, cnt = self._pairs_to_owners(a, dt)
            else:
                lid, val, cnt = None, None, torch.zeros(5, dtype=torch.float64, device=dev)
            got.append((lid, val))
            counts.append(cnt)
        pers_sum = got[0][1].to(torch.float64).sum().reshape(1) if given[0] else torch.zeros(1, dtype=torch.float64,
                                                                                               device=dev)
        tot = torch.cat(counts + [pers_sum])
        dist.all_reduce(tot)
        (pm, pn, pneg, pinv, pdup), (gm, _, _, ginv, _), (om, _, _, oinv, _) = [tot[5 * k:5 * k + 5].tolist() for k in range(3)]
        total_sum = float(tot[15].item())
        where = "MGGraph.pagerank"

        def fail(cls, code, message):
            raise cls(code, message, where)

        if given[0]:
            if pm:
                fail(capi.CugraphRuntimeError, capi.UNKNOWN_ERROR, "Invalid input argument: if personalization.has_value() is "
                     "true, the size of vertices and values should match")
            if pn == 0:
                fail(capi.CugraphRuntimeError, capi.UNKNOWN_ERROR, "Invalid input argument: if personalizations.has_value() "
                     "is true, the input personalization vector size should not be 0.")
            if pinv:
                fail(capi.CugraphValueError, capi.INVALID_INPUT,
                     "Invalid input argument: peresonalization vertices have invalid vertex IDs.")
            if pneg:
                fail(capi.CugraphValueError, capi.INVALID_INPUT,
                     "Invalid input argument: peresonalization values should be non-negative.")
            if pdup:
                fail(capi.CugraphValueError, capi.INVALID_INPUT,
                     "Invalid input argument: personalization vertices should not contain duplicate entries.")
            if not total_sum > 0.0:
                fail(capi.CugraphRuntimeError, capi.UNKNOWN_ERROR,
                     "Invalid input argument: sum of personalization valuese should be positive.")
        for k, name, mism, inv in ((1, "initial_guess", gm, ginv), (2, "precomputed_out_weights", om, oinv)):
            if given[k] and mism:
                fail(capi.CugraphValueError, capi.INVALID_INPUT, f"{name}: vertex and value arrays differ in size")
            if given[k] and inv:
                fail(capi.CugraphValueError, capi.INVALID_INPUT,
                     f"{name}: vertex list contains ids that are not vertices of the graph")
        dense = []
        for k, (lid, val) in enumerate(got):
            if not given[k]:
                dense.append(None)
                continue
            out = torch.zeros(mp, dtype=dt, device=dev)
            out[lid] = val
            dense.append(out)
        return dense[0], total_sum, dense[1], dense[2]

    # ------------------------------------------------------------------------------------------
    # multi-GPU BFS.  The reference's MG BFS (bfs_impl.cuh:446-869) moves the frontier through the edge partitions with
    # fill_edge_dst_property broadcasts (fill_edge_src_dst_property.cuh:1368) and an all-to-all-v of the discovered
    # (vertex, predecessor) pairs over the row communicator (transform_reduce_if_v_frontier_outgoing_e_by_dst.cuh:981-1074).
    # Here one level is: all-gather of the owners' frontier flags inside the column group (-> flags over the block's
    # source slots), all-gather of the visited flags inside the row group (-> flags over its destination slots), ONE step
    # on the block, ONE max-reduce-scatter of the candidate predecessors inside the row group, the owners' update and one
    # all-reduce of the new frontier's size (with its degree sums when the direction is chosen per level).  The step is
    # top-down (cugraph_b200_block_bfs_push: the frontier columns push their edges into the unvisited rows) or bottom-up
    # (cugraph_b200_block_bfs_pull: every unvisited row looks for a source in the frontier); both take and give the same
    # arrays, so the collectives of a level never depend on its direction.
    # Distances are the BFS levels (bit-exact vs single-GPU); a predecessor is any frontier neighbour, as in the reference.
    # ------------------------------------------------------------------------------------------
    def bfs(self, source, depth_limit=-1, compute_predecessors=True, *, direction_optimizing=False):
        """BFS from one source or from a set of sources.  Returns (vertices, distances, predecessors) of the vertices this
        rank owns: int32 distances (INT32_MAX = unreachable), predecessors as external ids (-1 = none), or None when not
        requested.
          source a Python / NumPy integer or a 0-d tensor: one external vertex id, the same value on every rank;
            ValueError on every rank when it is not a vertex.
          source a 1-D tensor or array: external ids given by THIS rank (possibly none; ranks may give different or
            overlapping ids).  The BFS starts from the union of every rank's ids, each at distance 0 without a predecessor,
            as cugraph_bfs does with several sources; with no id on any rank every vertex is unreached.  Every rank raises
            the same error (one all-reduce): TypeError for ids in a dtype other than the edge ids' on some rank,
            CugraphValueError for an id that is not a vertex.
          direction_optimizing: False runs every level top-down, as cugraph_bfs does.  True picks each level's direction
            by single GPU's rule and knobs (cugraph_b200_bfs_bottom_up, CUGRAPH_B200_BFS_ALPHA / _BETA) over global counts:
            the frontier's size and out-degree sum, the unvisited vertices and the sum of their in-degrees (the first call
            counts the degrees, see degrees()).  Unlike cugraph_bfs, True is accepted on every graph, directed ones
            included: the block stores its edges by destination, so its bottom-up step reads true in-edges, and whether
            an edge list is symmetric is not known here anyway.  Only the schedule depends on the flag: the distances are
            the same, the predecessors may differ (any frontier neighbour).
        Every rank must pass the same form, a scalar or an array, and the same direction_optimizing (not checked: the
        collectives would not match).  Sets last_bfs_stats = dict(levels, top_down, bottom_up): the levels run and how
        many ran in each direction."""
        p, g = self.part, self.part.groups
        dev, mp = self.device, p.maxpart
        imax = torch.iinfo(torch.int32).max
        dist_own = torch.full((mp,), imax, dtype=torch.int32, device=dev)
        pred_code = torch.full((mp,), -1, dtype=torch.int64, device=dev)
        visited = torch.zeros(mp, dtype=torch.uint8, device=dev)
        visited[p.n_local:] = 1                                  # padding slots never take part
        frontier = torch.zeros(mp, dtype=torch.uint8, device=dev)
        if _is_scalar(source):
            lid = self._source_lid(source, "bfs")
            if lid >= 0:
                dist_own[lid] = 0
                visited[lid] = 1
                frontier[lid] = 1
        else:
            lids = self._sources_to_owners(source)
            dist_own[lids] = 0
            visited[lids] = 1
            frontier[lids] = 1
        do = bool(direction_optimizing)
        if do:
            # (out, in)-degrees over the owned slots, 0 in the padding; the frontier's counts and the edge total
            self.degrees()
            deg = torch.zeros((2, mp), dtype=torch.int64, device=dev)
            deg[0, :p.n_local] = self._degrees[1]
            deg[1, :p.n_local] = self._degrees[0]
            head = torch.cat([frontier.sum().to(torch.int64).reshape(1), (deg * frontier).sum(1), deg[1].sum().reshape(1)])
            dist.all_reduce(head)
            n_f, m_f, m_vis_in, m_total = head.tolist()          # m_vis_in: the in-degree sum of the visited vertices
            n_vis, prev_n_f = n_f, 0
        f_cols = torch.zeros(self.n_cols, dtype=torch.uint8, device=dev)
        v_rows = torch.zeros(self.n_rows, dtype=torch.uint8, device=dev)
        cand = torch.full((self.n_rows,), -1, dtype=torch.int64, device=dev)
        cand_own = torch.full((mp,), -1, dtype=torch.int64, device=dev)
        level = n_bottom_up = 0
        bottom_up = False
        with _views(f_cols, v_rows, cand) as (vf, vv, vc):
            while depth_limit < 0 or level < depth_limit:
                if do:
                    bottom_up = bool(self.lib.cugraph_b200_bfs_bottom_up(self.handle.ptr, 1 if bottom_up else 0, n_f, prev_n_f,
                                                                         m_f, m_total - m_vis_in, p.n_global - n_vis))
                all_gather_into(f_cols, frontier, g.col_group)
                all_gather_into(v_rows, visited, g.row_group)
                step = "cugraph_b200_block_bfs_pull" if bottom_up else "cugraph_b200_block_bfs_push"
                self._call(step, self.block, vf.ptr, vv.ptr, mp, g.C, g.c, vc.ptr)
                reduce_scatter_into(cand_own, cand, g.row_group, op=dist.ReduceOp.MAX)
                new = (visited == 0) & (cand_own >= 0)
                level += 1
                n_bottom_up += int(bottom_up)
                dist_own[new] = level
                pred_code[new] = cand_own[new]
                visited |= new.to(torch.uint8)
                frontier = new.to(torch.uint8)
                if do:
                    counts = torch.cat([new.sum().to(torch.int64).reshape(1), (deg * new).sum(1)])
                    dist.all_reduce(counts)
                    n_new, m_new, in_new = counts.tolist()
                    prev_n_f, n_f, m_f = n_f, n_new, m_new
                    n_vis += n_new
                    m_vis_in += in_new
                else:
                    n_new = _global_count(new)
                if n_new == 0:
                    break
        self.last_bfs_stats = dict(levels=level, top_down=level - n_bottom_up, bottom_up=n_bottom_up)
        verts = p.vertices
        d_out = dist_own[:p.n_local].clone()
        if not compute_predecessors:
            return verts, d_out, None
        return verts, d_out, self._codes_to_external(pred_code[:p.n_local])

    def _source_lid(self, source, what):
        """local id of the external vertex `source` on this rank, -1 when another rank owns it; ValueError on every rank when
        it is not a vertex (one all-reduce)"""
        p, g = self.part, self.part.groups
        owner = int(vertex_owner(torch.tensor([int(source)], dtype=torch.int64), g.world)[0])
        found = torch.zeros(1, dtype=torch.int64, device=self.device)
        lid = -1
        if owner == g.rank:
            hit = (p.vertices == int(source)).nonzero()
            if hit.numel():
                lid = int(hit[0, 0])
                found += 1
        dist.all_reduce(found)
        if int(found.item()) == 0:
            raise ValueError(f"{what} source {source} is not a vertex of the graph")
        return lid

    def _sources_to_owners(self, sources, where="MGGraph.bfs"):
        """the local ids of the sources, from every rank, that this rank owns (duplicates kept): each rank's ids travel to
        their owners in one all-to-all-v; one all-reduce of the error counts, and every rank raises the same error"""
        from cugraph_b200 import _capi as capi
        p, g, dev = self.part, self.part.groups, self.device
        s = torch.as_tensor(sources)
        bad_type = int(s.dtype != p.vertices.dtype)
        s = s.to(dev).reshape(-1).to(torch.int64) if not bad_type else torch.zeros(0, dtype=torch.int64, device=dev)
        (req,), _, _, _ = exchange([s], vertex_owner(s, g.world), g.world)
        lid, hit = self._owned_lids(req)
        errs = torch.stack([torch.tensor(bad_type, dtype=torch.int64, device=dev), (~hit).sum().to(torch.int64)])
        dist.all_reduce(errs)
        bad_type, invalid = errs.tolist()
        if bad_type:
            raise TypeError(f"{where}: sources must have the dtype of the edge ids on every rank")
        if invalid:
            raise capi.CugraphValueError(capi.INVALID_INPUT, "Found invalid vertex in the input sources", where)
        return lid

    # ------------------------------------------------------------------------------------------
    # multi-GPU multi-source BFS: one BFS per source, a batch of up to 64 sources per level (single GPU's bit-parallel BFS,
    # cugraph_b200_multi_source_bfs, on the partition).  The owners keep three INT64 words per owned slot, bit j for source j
    # of the batch: seen (reached), cur (reached at this level) and the received partials of next.  One level: all-gather of
    # cur inside the column group (-> the block's column slots) and of seen inside the row group (-> its row slots), ONE block
    # step (cugraph_b200_block_ms_bfs_push or _pull: the same arrays in and out) writing a partial next word per row slot, ONE
    # all-to-all of the partials inside the row group (NCCL has no bitwise reduce-scatter: each member receives the C slices
    # of its own slots and the owner step ORs them, the bytes of a reduce-scatter), the owner step
    # (cugraph_b200_ms_bfs_owner_step: new bits, distances, counts) and ONE all-reduce of the counts, which is also the
    # termination test.  With predecessors a level adds an all-gather of the new words inside the row group, the block's
    # predecessor step (cugraph_b200_block_ms_bfs_pred) into a pair buffer sized from the counts already read, ONE MAX
    # reduce-scatter of it, and the owners' scatter into the predecessor rows (cugraph_b200_ms_bfs_owner_pred).  The
    # predecessor of v in row k is the largest code among v's in-neighbours that source k reached one level earlier: what
    # the top-down MGGraph.bfs(sources[k]) keeps, whichever direction the batch's levels run.
    # ------------------------------------------------------------------------------------------
    def multi_source_bfs(self, sources, depth_limit=-1, compute_predecessors=True, *, direction_optimizing=False):
        """BFS from each of the sources separately.  sources: a 1-D tensor or array of external ids in the edge ids' dtype,
        the SAME list in the same order on every rank (source k names row k of the result); duplicates each get their own
        row.  Returns (vertices, distances, predecessors) of the vertices this rank owns: distances int32 [n, n_local]
        (INT32_MAX = unreached), predecessors [n, n_local] external ids in the vertices' dtype (-1 = none), or None when not
        requested.  Row k equals MGGraph.bfs(sources[k], depth_limit) on the same graph and grid: the same distances, and the
        predecessors of its default top-down schedule.  The sources run in batches of 64.
          direction_optimizing: False runs every level top-down; True picks each level's direction by Beamer's rule
            (cugraph_b200_bfs_bottom_up) over global counts, a vertex counting as visited once every source of the batch
            has reached it, with its in-degree for the unvisited edges (as MGGraph.bfs counts them).  Only the schedule
            depends on it.
        Every rank raises the same error: TypeError for sources in a dtype other than the edge ids' on some rank,
        ValueError when the lists differ between ranks, CugraphValueError for a source that is not a vertex.  Sets
        last_ms_bfs_stats = dict(batches, levels, top_down, bottom_up), the levels summed over the batches."""
        p = self.part
        lids = self._ms_sources(sources)
        n, n_loc = lids.numel(), p.n_local
        dist_out = torch.full((n, n_loc), torch.iinfo(torch.int32).max, dtype=torch.int32, device=self.device)
        pred_out = torch.full((n, n_loc), -1, dtype=p.vertices.dtype, device=self.device) if compute_predecessors else None
        deg = None
        if direction_optimizing:
            self.degrees()
            deg = (self._degrees[1].to(torch.int64), self._degrees[0].to(torch.int64))   # (out, in)
        stats = dict(batches=0, levels=0, top_down=0, bottom_up=0)
        for b0 in range(0, n, 64):
            nb = min(64, n - b0)
            codes = self._ms_bfs_batch(lids[b0:b0 + nb], dist_out[b0:b0 + nb], depth_limit, compute_predecessors, deg, stats)
            if compute_predecessors:   # one batch of int64 codes alive at a time, its exchange in pieces of <= 2^27 codes
                step = max(1, (1 << 27) // p.maxpart)          # the same on every rank: each piece is a collective
                for k0 in range(0, nb, step):
                    k1 = min(k0 + step, nb)
                    pred_out[b0 + k0:b0 + k1] = self._codes_to_external(codes[k0 * n_loc:k1 * n_loc]).reshape(k1 - k0, n_loc)
        self.last_ms_bfs_stats = stats
        return p.vertices, dist_out, pred_out

    def _ms_sources(self, sources):
        """multi_source_bfs's source list -> the local id of every source on this rank, -1 where another rank owns it.  Two
        MAX all-reduces check that every rank has the same list: [n, -n, dtype error], then [ids, -ids, invalid]; a list
        that differs at some position shows there as max != -max(-x) on every rank."""
        from cugraph_b200 import _capi as capi
        p, g, dev = self.part, self.part.groups, self.device
        where = "MGGraph.multi_source_bfs"
        s = torch.as_tensor(sources)
        bad_type = int(s.dtype != p.vertices.dtype)
        s = s.to(dev).reshape(-1).to(torch.int64)
        n = s.numel()
        head = torch.tensor([n, -n, bad_type], dtype=torch.int64, device=dev)
        dist.all_reduce(head, op=dist.ReduceOp.MAX)
        n_max, n_min_neg, bad_type = head.tolist()
        if bad_type:
            raise TypeError(f"{where}: sources must have the dtype of the edge ids on every rank")
        if n_max != -n_min_neg:
            raise ValueError(f"{where}: sources must be the same list, in the same order, on every rank")
        if n == 0:
            return torch.zeros(0, dtype=torch.int64, device=dev)
        lid, hit = self._owned_lids(s)
        invalid = ((vertex_owner(s, g.world) == g.rank) & ~hit).sum().reshape(1)   # every id has one owner to check it
        chk = torch.cat([s, -s, invalid])
        dist.all_reduce(chk, op=dist.ReduceOp.MAX)
        if bool(((chk[:n] != s) | (chk[n:2 * n] != -s)).any()):
            raise ValueError(f"{where}: sources must be the same list, in the same order, on every rank")
        if int(chk[2 * n].item()):
            raise capi.CugraphValueError(capi.INVALID_INPUT, "Found invalid vertex in the input sources", where)
        return torch.where(hit, lid, -1)

    def _ms_bfs_batch(self, lids, dist_rows, depth_limit, want_pred, deg, stats):
        """one batch of nb <= 64 sources (their local ids here, -1 elsewhere): fills dist_rows [nb, n_local] and returns the
        predecessor codes (nb * n_local, -1 = none) or None"""
        p, g, dev, mp = self.part, self.part.groups, self.device, self.part.maxpart
        n_loc, nb, i64 = p.n_local, lids.numel(), torch.int64
        mask = -1 if nb == 64 else (1 << nb) - 1
        seen = torch.zeros(mp, dtype=i64, device=dev)
        seen[n_loc:] = mask                                   # padding slots never take part
        mine = (lids >= 0).nonzero().reshape(-1)              # the batch positions whose source this rank owns
        ml = lids[mine]
        seen.index_put_((ml,), torch.bitwise_left_shift(torch.ones_like(mine), mine), accumulate=True)  # distinct bits: sum = OR
        cur = torch.zeros(mp, dtype=i64, device=dev)
        cur[:n_loc] = seen[:n_loc]
        dist_rows[mine, ml] = 0
        do = deg is not None
        if do:
            u = torch.unique(ml)
            full = seen[u] == mask
            head = torch.stack([torch.tensor(u.numel(), device=dev), deg[0][u].sum(), full.sum(), deg[1][u[full]].sum(),
                                deg[1].sum()]).to(i64)
            dist.all_reduce(head)
            n_f, m_f, n_full, in_full, m_total = head.tolist()
            prev_n_f = 0
        cur_cols = torch.empty(self.n_cols, dtype=i64, device=dev)
        seen_rows = torch.empty(self.n_rows, dtype=i64, device=dev)
        next_rows = torch.empty(self.n_rows, dtype=i64, device=dev)
        recv = next_rows if g.C == 1 else torch.empty(self.n_rows, dtype=i64, device=dev)   # C slices of maxpart
        counts = torch.zeros(5, dtype=i64, device=dev)
        tot = torch.zeros(4 + g.world, dtype=i64, device=dev)   # the four counts, then every rank's new bits
        codes = torch.full((nb * n_loc,), -1, dtype=i64, device=dev) if want_pred else None
        new_rows = torch.empty(self.n_rows, dtype=i64, device=dev) if want_pred else None
        d_out, d_in = deg if do else (None, None)
        level = n_bottom_up = 0
        bottom_up = False
        with _views(cur_cols, seen_rows, next_rows, recv, seen, cur, dist_rows.reshape(-1), d_out, d_in, counts, new_rows,
                    codes) as (vcc, vsr, vnr, vrc, vs, vc, vd, vdo, vdi, vk, vnw, vcode):
            while depth_limit < 0 or level < depth_limit:
                if do:
                    bottom_up = bool(self.lib.cugraph_b200_bfs_bottom_up(self.handle.ptr, 1 if bottom_up else 0, n_f, prev_n_f,
                                                                         m_f, m_total - in_full, p.n_global - n_full))
                all_gather_into(cur_cols, cur, g.col_group)
                all_gather_into(seen_rows, seen, g.row_group)
                step = "cugraph_b200_block_ms_bfs_pull" if bottom_up else "cugraph_b200_block_ms_bfs_push"
                self._call(step, self.block, vcc.ptr, vsr.ptr, nb, vnr.ptr)
                if g.C > 1:
                    dist.all_to_all_single(recv, next_rows, group=g.row_group)
                level += 1
                n_bottom_up += int(bottom_up)
                self._call("cugraph_b200_ms_bfs_owner_step", vrc.ptr, g.C, mp, n_loc, nb, level, vs.ptr, vc.ptr, vd.ptr, vdo.ptr,
                           vdi.ptr, vk.ptr)
                tot.zero_()
                tot[:4] = counts[:4]
                tot[4 + g.rank] = counts[4]
                dist.all_reduce(tot)
                t = tot.tolist()
                n_new = t[0]
                # the row group's pair buffer: C segments, each as long as the most new bits one member owns
                seg = max(t[4 + g.r * g.C + k] for k in range(g.C)) if want_pred else 0
                if seg:
                    all_gather_into(new_rows, cur, g.row_group)
                    pairs = torch.empty(g.C * seg, dtype=i64, device=dev)
                    pairs_own = torch.empty(seg, dtype=i64, device=dev)
                    with _views(pairs) as (vp,):
                        self._call("cugraph_b200_block_ms_bfs_pred", self.block, vcc.ptr, vnw.ptr, mp, g.C, g.c, seg, vp.ptr)
                    reduce_scatter_into(pairs_own, pairs, g.row_group, op=dist.ReduceOp.MAX)
                    with _views(pairs_own) as (vpo,):
                        self._call("cugraph_b200_ms_bfs_owner_pred", vc.ptr, vpo.ptr, n_loc, nb, vcode.ptr)
                if do:
                    prev_n_f, n_f, m_f = n_f, n_new, t[1]
                    n_full += t[2]
                    in_full += t[3]
                if n_new == 0:
                    break
        stats["batches"] += 1
        stats["levels"] += level
        stats["top_down"] += level - n_bottom_up
        stats["bottom_up"] += n_bottom_up
        return codes

    def _codes_to_external(self, codes):
        """predecessor codes (owner rank * maxpart + local id, -1 = none) -> external ids, answered by the owners (one
        all-to-all-v there and back)"""
        p, g, dev, mp = self.part, self.part.groups, self.device, self.part.maxpart
        verts = p.vertices
        has = codes >= 0
        ask = codes[has]
        (req,), order, sc, rc = exchange([ask % mp], torch.div(ask, mp, rounding_mode="floor"), g.world)
        ans = verts[req]
        back = torch.empty(sum(sc), dtype=ans.dtype, device=dev)
        dist.all_to_all_single(back, ans.contiguous(), output_split_sizes=sc, input_split_sizes=rc)
        got = torch.empty_like(back)
        got[order] = back
        pred = torch.full((codes.numel(),), -1, dtype=verts.dtype, device=dev)
        pred[has] = got
        return pred

    # ------------------------------------------------------------------------------------------
    # multi-GPU extract_paths: single GPU's walk (k_paths_max_len / k_paths_walk, traverse.cu) spread over the owners, one
    # path position per round, as the reference gathers one position per round over all destinations
    # (extract_bfs_paths_impl.cuh:129-238).  Set-up, once per call: the owned predecessors become codes (owner rank * maxpart
    # + local id; one all-to-all-v to their owners and back, the inverse of _codes_to_external); every destination asks its
    # owner for (distance, predecessor code) (one all-to-all-v there and back); ONE MAX all-reduce gives max_path_length;
    # cugraph_b200_paths_advance writes every destination into its own column and groups the walks that go on by the owner
    # of their next vertex.  Then exactly max_path_length - 1 rounds on every rank, a fixed count that needs no termination
    # all-reduce.  One round: an all-to-all of the per-rank request counts (read back together with the counts sent), an
    # all-to-all-v of the requested local ids to their owners, cugraph_b200_paths_answer there, an all-to-all-v of the
    # (external id, predecessor code) answers back in request order, and cugraph_b200_paths_advance.
    # ------------------------------------------------------------------------------------------
    def extract_paths(self, distances, predecessors, destinations):
        """Paths from the BFS sources to `destinations` (single-GPU cugraph_extract_paths' semantics).  distances (int32) and
        predecessors (external ids) are the n_local entries MGGraph.bfs returned on this rank; destinations are external ids
        given by this rank, any ids (owned by any rank, or not vertices at all), possibly none.  Returns (paths,
        max_path_length): paths[i] ([len(destinations), max_path_length], the vertices' dtype) holds the path from the source
        to destinations[i] in columns 0 .. distance, -1 elsewhere; a source gives [source, -1, ...]; an unreached destination,
        an id that is not a vertex, or a distance >= max_path_length gives a row of -1; a predecessor that is not a vertex ends
        the walk.  max_path_length = 1 + the largest distance among the destinations of EVERY rank that have a predecessor
        (the same on every rank).  Every rank raises the same error (one all-reduce): ValueError when distances or
        predecessors do not hold n_local entries (or are None), or a rank has 2^31 or more destinations; TypeError for
        distances that are not int32.  Sets last_paths_stats = dict(rounds)."""
        p, g, dev, mp = self.part, self.part.groups, self.device, self.part.maxpart
        n, P = p.n_local, g.world
        imax = torch.iinfo(torch.int32).max
        dst = torch.as_tensor(destinations).to(dev).reshape(-1).to(torch.int64)
        m = dst.numel()
        if distances is not None:
            distances = torch.as_tensor(distances).to(dev).reshape(-1)
        if predecessors is not None:
            predecessors = torch.as_tensor(predecessors).to(dev).reshape(-1)
        bad_size = int(distances is None or predecessors is None or distances.numel() != n or predecessors.numel() != n
                       or m > imax)
        bad_type = int(not bad_size and distances.dtype != torch.int32)
        errs = torch.tensor([bad_size, bad_type], dtype=torch.int64, device=dev)
        dist.all_reduce(errs)
        bad_size, bad_type = errs.tolist()
        if bad_size:
            raise ValueError("MGGraph.extract_paths: distances and predecessors must be the n_local entries MGGraph.bfs "
                             "returned on every rank, and each rank may give fewer than 2^31 destinations")
        if bad_type:
            raise TypeError("MGGraph.extract_paths: distances must be int32 on every rank")
        # owned predecessors -> codes, answered by the predecessors' owners (-1: none, or not a vertex)
        pred = predecessors.to(torch.int64)
        has = pred != -1
        ask = pred[has]
        (req,), order, sc, rc = exchange([ask], vertex_owner(ask, P), P)
        lid, hit = self._owned_lids(req)
        ans = torch.where(hit, g.rank * mp + lid, -1)
        back = torch.empty(sum(sc), dtype=torch.int64, device=dev)
        dist.all_to_all_single(back, ans, output_split_sizes=sc, input_split_sizes=rc)
        got = torch.empty_like(back)
        got[order] = back
        pred_code = torch.full((n,), -1, dtype=torch.int64, device=dev)
        pred_code[has] = got
        # destinations -> (distance, predecessor code) from their owners; INT32_MAX / -1 for an id that is not a vertex
        d_own = distances.to(torch.int64)
        (req,), order, sc, rc = exchange([dst], vertex_owner(dst, P), P)
        lid, hit = self._owned_lids(req)
        ans = torch.full((req.numel(), 2), -1, dtype=torch.int64, device=dev)
        ans[:, 0] = imax
        ans[hit, 0] = d_own[lid[hit]]
        ans[hit, 1] = pred_code[lid[hit]]
        back = torch.empty(2 * sum(sc), dtype=torch.int64, device=dev)
        dist.all_to_all_single(back, ans.reshape(-1), output_split_sizes=[2 * k for k in sc],
                               input_split_sizes=[2 * k for k in rc])
        got = torch.empty((m, 2), dtype=torch.int64, device=dev)
        got[order] = back.view(-1, 2)
        d_dst, c_dst = got[:, 0], got[:, 1]
        mx = torch.zeros(1, dtype=torch.int64, device=dev)
        if m:
            mx = torch.maximum(mx, torch.where((d_dst < imax) & (c_dst >= 0), d_dst, 0).max())
        dist.all_reduce(mx, op=dist.ReduceOp.MAX)
        length = int(mx.item()) + 1
        paths = torch.full((m, length), -1, dtype=p.vertices.dtype, device=dev)
        rows = ((d_dst >= 0) & (d_dst < length)).nonzero().reshape(-1)
        answers = torch.stack([dst[rows], c_dst[rows]], 1).reshape(-1)
        cap = max(rows.numel(), 1)       # a walk never splits: no round has more entries than the first
        cur = [rows.to(torch.int32), d_dst[rows].to(torch.int32)]
        bufs = [[torch.empty(cap, dtype=torch.int32, device=dev) for _ in range(3)] for _ in range(2)]
        counts = torch.empty(2 * P, dtype=torch.int64, device=dev)   # [sent to each rank, received from each rank]

        def advance(answers, rows, pos, nxt):
            with _views(answers, rows, pos, paths.view(-1), *nxt, counts) as vs:
                self._call("cugraph_b200_paths_advance", *[v.ptr for v in vs[:4]], length, mp, P, *[v.ptr for v in vs[4:]])

        advance(answers, cur[0], cur[1], bufs[0])
        for k in range(length - 1):
            lids_out, rows_k, pos_k = bufs[k % 2]
            dist.all_to_all_single(counts[P:], counts[:P])
            both = counts.tolist()
            sc, rc = both[:P], both[P:]
            ns, nr = sum(sc), sum(rc)
            lids_in = torch.empty(nr, dtype=torch.int32, device=dev)
            dist.all_to_all_single(lids_in, lids_out[:ns], output_split_sizes=rc, input_split_sizes=sc)
            answers = torch.empty(2 * nr, dtype=torch.int64, device=dev)
            with _views(lids_in, p.vertices, pred_code, answers) as (vl, vv, vc, va):
                self._call("cugraph_b200_paths_answer", vl.ptr, vv.ptr, vc.ptr, n, va.ptr)
            back = torch.empty(2 * ns, dtype=torch.int64, device=dev)
            dist.all_to_all_single(back, answers, output_split_sizes=[2 * x for x in sc], input_split_sizes=[2 * x for x in rc])
            advance(back, rows_k[:ns], pos_k[:ns], bufs[(k + 1) % 2])
        self.last_paths_stats = dict(rounds=length - 1)
        return paths, length

    # ------------------------------------------------------------------------------------------
    # multi-GPU SSSP.  The reference's MG SSSP (sssp_impl.cuh:301-375) gathers the distances of the frontier's sources over
    # the edge partitions (update_edge_src_property) and reduces the proposals per destination to the owners.  Here the
    # owners keep dist / pred_code / pending (improved, not relaxed yet) for their vertices, and the rounds run inside
    # Δ-windows [lo, hi) over the distance range.  One round: the pending vertices below hi are the frontier; their distances
    # (+inf for everybody else) are all-gathered inside the column group over the block's source slots; the block relaxes
    # their edges into one INT64 key per destination slot (cugraph_b200_block_sssp_relax: float = distance bits << 32 | code
    # of the source, double = distance bits); ONE MIN reduce-scatter inside the row group brings the smallest key to the
    # owner, who accepts strict improvements only.  Double runs with predecessors take a second exchange for the codes
    # (cugraph_b200_block_sssp_pred).  Strict improvement with the "smallest distance, then smallest code" order keeps the
    # predecessors a tree, also through zero-weight cycles.  Distances are the fixpoint of float add / min: bit-exact vs one GPU
    # whatever Δ is.  Δ follows the single-GPU controller (DESIGN §3.4): the reference's 32 * avg weight / avg degree
    # (sssp_impl.cuh:246-247) / 64 at the start, x2 after a window of <= 2 rounds, / 2 after one of >= 6;
    # CUGRAPH_B200_MG_SSSP_DELTA_SCALE multiplies it (results never depend on it).
    # ------------------------------------------------------------------------------------------
    def _sssp_delta(self):
        if self._sssp_avg is None:   # global averages, one all-reduce at the first call
            t = torch.tensor([self._w_sum_local, float(self.num_edges_local)], dtype=torch.float64, device=self.device)
            dist.all_reduce(t)
            w_sum, n_edges = t.tolist()
            avg_w = w_sum / n_edges if n_edges > 0 else 0.0
            self._sssp_avg = (avg_w, n_edges / max(self.part.n_global, 1))
        avg_w, avg_deg = self._sssp_avg
        ref = 32.0 * avg_w / max(avg_deg, 1e-30) * float(os.environ.get("CUGRAPH_B200_MG_SSSP_DELTA_SCALE", "1"))
        if not ref > 0.0 or math.isinf(ref):
            ref = 1.0
        return ref / 64.0, ref / 4096.0

    def sssp(self, source, cutoff=math.inf, compute_predecessors=True):
        """source: external vertex id (the same value on every rank).  Returns (vertices, distances, predecessors) of the
        vertices this rank owns: distances in the weight dtype (FLT_MAX / DBL_MAX = unreachable, the reference's convention,
        sssp_impl.cuh:215-229), predecessors as external ids (-1 = none), or None when not requested."""
        if not self.weighted:
            raise ValueError("SSSP requires a weighted graph")
        p, g = self.part, self.part.groups
        dev, dt, mp = self.device, self.dtype, p.maxpart
        f32 = dt == torch.float32
        lid = self._source_lid(source, "sssp")
        inf = torch.tensor(math.inf, dtype=dt, device=dev)
        dist_own = torch.full((mp,), torch.finfo(dt).max, dtype=dt, device=dev)
        pred_code = torch.full((mp,), -1, dtype=torch.int64, device=dev)
        pending = torch.zeros(mp, dtype=torch.bool, device=dev)
        if lid >= 0:
            dist_own[lid] = 0
            pending[lid] = True
        delta, delta_floor = self._sssp_delta()
        want_codes = compute_predecessors and not f32
        x_cols = torch.empty(self.n_cols, dtype=dt, device=dev)
        cand = torch.empty(self.n_rows, dtype=torch.int64, device=dev)
        cand_own = torch.empty(mp, dtype=torch.int64, device=dev)
        win_rows = code_rows = None
        if want_codes:
            win_rows = torch.empty(self.n_rows, dtype=dt, device=dev)
            code_rows = torch.empty(self.n_rows, dtype=torch.int64, device=dev)
            code_own = torch.empty(mp, dtype=torch.int64, device=dev)
        hi = window_bound(0.0, delta, dt, dev)
        rounds = windows = window_rounds = 0
        with _views(x_cols, cand, win_rows, code_rows) as (vx, vc, vw, vk):
            while True:
                active = pending & (dist_own < hi)
                if _global_count(active) == 0:   # the window is done: open the next one at the smallest pending distance
                    windows += 1
                    if window_rounds <= 2:
                        delta = delta * 2.0 if delta < torch.finfo(dt).max / 4 else delta
                    elif window_rounds >= 6 and delta > delta_floor:
                        delta = delta / 2.0
                    m = torch.where(pending, dist_own, inf).min().view(1)
                    dist.all_reduce(m, op=dist.ReduceOp.MIN)
                    lo = float(m.item())
                    if math.isinf(lo):
                        break
                    hi = window_bound(lo, delta, dt, dev)
                    window_rounds = 0
                    continue
                pending &= ~active
                x = torch.where(active, dist_own, inf)
                all_gather_into(x_cols, x, g.col_group)              # partition-major = the block's column order
                self._call("cugraph_b200_block_sssp_relax", self.block, vx.ptr, float(cutoff), mp, g.C, g.c, vc.ptr)
                reduce_scatter_into(cand_own, cand, g.row_group, op=dist.ReduceOp.MIN)
                improved = sssp_owner_step(dist_own, pred_code, pending, cand_own)
                if want_codes:
                    all_gather_into(win_rows, torch.where(improved, dist_own, inf), g.row_group)
                    self._call("cugraph_b200_block_sssp_pred", self.block, vx.ptr, vw.ptr, mp, g.C, g.c, vk.ptr)
                    reduce_scatter_into(code_own, code_rows, g.row_group, op=dist.ReduceOp.MIN)
                    pred_code.copy_(torch.where(improved, code_own, pred_code))
                rounds += 1
                window_rounds += 1
        self.last_sssp_stats = dict(rounds=rounds, windows=windows)
        verts = p.vertices
        d_out = dist_own[:p.n_local].clone()
        if not compute_predecessors:
            return verts, d_out, None
        return verts, d_out, self._codes_to_external(pred_code[:p.n_local])

    # ------------------------------------------------------------------------------------------
    # BFS / SSSP certificate (validate_bfs, validate_sssp): the checks of a Graph500 validation, distributed over the same
    # edge block the traversals use, so that a result of any size on any grid is checked without gathering it.  Each rank
    # gives any set of (external id, distance, predecessor id) triples.  One all-to-all-v brings them to their owners, one
    # all-to-all-v there and back turns the predecessor ids into codes (owner rank * maxpart + local id, the inverse of
    # _codes_to_external).  The owners' distances are all-gathered over the block's column slots (column group) and its
    # row slots (row group), the predecessor codes over its row slots; ONE push round over the block's column-major copy
    # (cugraph_b200_block_check_paths) counts the edges that could still shorten a distance and marks every row whose
    # predecessor edge attains its distance (2 for a flat edge, d[p] = d[v]); ONE MAX reduce-scatter brings the marks to
    # the owners, whose per-vertex rules are torch passes.  SSSP predecessors can close a cycle only over flat edges: when
    # some exist, pointer jumping over them (an all-to-all-v there and back per round, as extract_paths walks) finds the
    # vertices whose chain never leaves them.  One all-reduce of the counters gives every rank the same verdict.
    # ------------------------------------------------------------------------------------------
    def validate_bfs(self, vertices, distances, predecessors, sources, depth_limit=-1):
        """Check a BFS result on this graph: returns a dict, the same on every rank, with `ok` and one count per rule
        (see _validate): not_vertex, missing, duplicate, bad_value, root, unreached, edge, tree_edge, cycle (always 0 for
        BFS), and edges_from_reached (stored edges whose source is reached; for a graph that stores both directions of
        every input edge, twice the input edges of the sources' component).  vertices, distances (int32, INT32_MAX =
        unreached) and predecessors (external ids, -1 = none) are this rank's triples, any of them, in any order: what
        MGGraph.bfs returned, or on a 1x1 grid a whole single-GPU cugraph_bfs result.  sources takes both forms bfs
        accepts; depth_limit as in bfs.  Every rank raises the same error: ValueError for arrays of unequal length or
        predecessors=None, TypeError for ids in another dtype than the edge ids' or distances that are not int32, and the
        errors of bfs for the sources.  No input is modified."""
        return self._validate(True, vertices, distances, predecessors, sources, depth_limit=depth_limit)

    def validate_sssp(self, vertices, distances, predecessors, source, cutoff=math.inf):
        """Check an SSSP result on this graph, as validate_bfs checks a BFS result: distances in the graph's weight dtype
        (finfo.max = unreached), `source` one external id (the same on every rank), cutoff as in sssp.  Predecessors must
        form no cycle (`cycle` counts the vertices whose predecessor chain runs into one).  ValueError on an unweighted
        graph."""
        if not self.weighted:
            raise ValueError("SSSP requires a weighted graph")
        return self._validate(False, vertices, distances, predecessors, source, cutoff=cutoff)

    def _validate(self, bfs, vertices, distances, predecessors, sources, depth_limit=-1, cutoff=math.inf):
        """The rules (d = distance, p = predecessor, unreached = the sentinel):
          not_vertex, missing, duplicate: every given id is a vertex; every vertex is given exactly once over all ranks.
          bad_value: d lies in [0, sentinel] and is not NaN (a bad value then counts as unreached).
          root: BFS, v is a source <=> d = 0 and p = -1; SSSP, the source has d = 0 and p = -1.
          unreached: a vertex other than a source is unreached <=> p = -1.
          edge: every stored edge u -> v with u reached and the step allowed has d[v] <= d[u] + 1 (BFS) or d[v] <= d[u] + w
            (SSSP, added in the weight dtype).  Allowed: BFS, depth_limit < 0 or d[u] < depth_limit; SSSP, d[u] + w below
            the cutoff rounded to the weight dtype (the arithmetic of the relaxation).
          tree_edge: every v with p != -1 has a stored edge p -> v with p reached, the step allowed and d[v] = d[p] + 1
            (BFS) or d[p] + w exactly (SSSP).
          cycle (SSSP): the predecessors form no cycle."""
        p, g, dev, mp = self.part, self.part.groups, self.device, self.part.maxpart
        P, n = g.world, p.n_local
        i64 = torch.int64
        ddt = torch.int32 if bfs else self.dtype
        vdt = p.vertices.dtype
        unreached = torch.iinfo(torch.int32).max if bfs else torch.finfo(ddt).max
        flat_t = lambda a: None if a is None else torch.as_tensor(a).to(dev).reshape(-1)  # noqa: E731
        v_in, d_in, p_in = flat_t(vertices), flat_t(distances), flat_t(predecessors)
        bad_size = int(v_in is None or d_in is None or p_in is None or not v_in.numel() == d_in.numel() == p_in.numel())
        bad_ids = int(not bad_size and (v_in.dtype != vdt or p_in.dtype != vdt))
        bad_dist = int(not bad_size and d_in.dtype != ddt)
        errs = torch.tensor([bad_size, bad_ids, bad_dist], dtype=i64, device=dev)
        dist.all_reduce(errs)
        bad_size, bad_ids, bad_dist = errs.tolist()
        where = "MGGraph.validate_bfs" if bfs else "MGGraph.validate_sssp"
        if bad_size:
            raise ValueError(f"{where}: vertices, distances and predecessors must be given, with equal lengths, on every rank")
        if bad_ids:
            raise TypeError(f"{where}: vertices and predecessors must have the dtype of the edge ids on every rank")
        if bad_dist:
            raise TypeError(f"{where}: distances must be {str(ddt)[6:]} on every rank")
        is_src = torch.zeros(mp, dtype=torch.bool, device=dev)
        if bfs and not _is_scalar(sources):
            is_src[self._sources_to_owners(sources, where)] = True
        else:
            lid = self._source_lid(sources, "validate_bfs" if bfs else "validate_sssp")
            if lid >= 0:
                is_src[lid] = True
        # the triples -> their owners
        vid = v_in.to(i64)
        (rv, rd, rp), _, _, _ = exchange([vid, d_in, p_in.to(i64)], vertex_owner(vid, P), P)
        lid, hit = self._owned_lids(rv)
        n_not_vertex = (~hit).sum()
        lid, rd, rp = lid[hit], rd[hit], rp[hit]
        cnt = torch.bincount(lid, minlength=mp)
        n_dup = (cnt - 1).clamp(min=0).sum()
        given = cnt > 0
        n_missing = (~given[:n]).sum()
        bad = rd < 0 if bfs else torch.isnan(rd) | (rd < 0) | (rd > unreached)
        d_own = torch.full((mp,), unreached, dtype=ddt, device=dev)
        d_own[lid] = torch.where(bad, torch.full_like(rd, unreached), rd)
        pext = torch.full((mp,), -1, dtype=i64, device=dev)
        pext[lid] = rp
        # predecessor ids -> codes, answered by their owners (-2: not a vertex)
        has = pext != -1
        ask = pext[has]
        (req,), order, sc, rc = exchange([ask], vertex_owner(ask, P), P)
        l2, h2 = self._owned_lids(req)
        ans = torch.where(h2, g.rank * mp + l2, -2)
        back = torch.empty(sum(sc), dtype=i64, device=dev)
        dist.all_to_all_single(back, ans, output_split_sizes=sc, input_split_sizes=rc)
        code = torch.full((mp,), -1, dtype=i64, device=dev)
        code[has] = _unpermute(back, order)
        # the edge rules on the block
        reached = given & (d_own != unreached)
        d_act = d_own if bfs else torch.where(reached, d_own, torch.tensor(math.inf, dtype=ddt, device=dev))
        d_cols = torch.empty(self.n_cols, dtype=ddt, device=dev)
        d_rows = torch.empty(self.n_rows, dtype=ddt, device=dev)
        c_rows = torch.empty(self.n_rows, dtype=i64, device=dev)
        all_gather_into(d_cols, d_act, g.col_group)
        all_gather_into(d_rows, d_own, g.row_group)
        all_gather_into(c_rows, code, g.row_group)
        flags = torch.empty(self.n_rows, dtype=torch.uint8, device=dev)
        viol = torch.zeros(1, dtype=i64, device=dev)
        edges = C.c_uint64(0)
        lim = (float(depth_limit) + 1.0 if depth_limit >= 0 else math.inf) if bfs else float(cutoff)
        with _views(d_cols, d_rows, c_rows, flags, viol) as (vc, vr, vp, vf, vv):
            self._call("cugraph_b200_block_check_paths", self.block, vc.ptr, vr.ptr, vp.ptr, lim, mp, g.C, g.c, vf.ptr, vv.ptr,
                       C.byref(edges))
        flag = torch.empty(mp, dtype=torch.uint8, device=dev)
        reduce_scatter_into(flag, flags, g.row_group, op=dist.ReduceOp.MAX)
        # the per-vertex rules at the owners
        gv, dv, cv, sv, fv = given[:n], d_own[:n], code[:n], is_src[:n], flag[:n]
        zero_root = (dv == 0) & (cv == -1)
        root = gv & (sv != zero_root) if bfs else gv & sv & ~zero_root
        unreach = gv & ~sv & ((dv == unreached) != (cv == -1))
        tree = gv & (cv != -1) & (fv == 0)
        n_cycle = torch.zeros((), dtype=i64, device=dev)
        if not bfs:
            flat = torch.zeros(mp, dtype=torch.bool, device=dev)
            flat[:n] = gv & (cv >= 0) & (fv == 2)
            n_flat = _global_count(flat)
            if n_flat:
                n_cycle = self._flat_cycles(flat, code, n_flat)
        counts = torch.stack([n_not_vertex, n_missing, n_dup, bad.sum(), root.sum(), unreach.sum(), viol[0], tree.sum(),
                              n_cycle, torch.tensor(edges.value, device=dev)]).to(i64)
        dist.all_reduce(counts)
        names = ("not_vertex", "missing", "duplicate", "bad_value", "root", "unreached", "edge", "tree_edge", "cycle",
                 "edges_from_reached")
        out = dict(zip(names, counts.tolist()))
        out["ok"] = not any(out[k] for k in names[:-1])
        return out

    def _flat_cycles(self, flat, code, n_flat):
        """the vertices, over all ranks, whose predecessor chain through flat tree edges never ends: pointer jumping (each
        round: every unfinished vertex asks the owner of its pointer for that vertex's pointer and whether it is finished,
        an all-to-all-v there and back, then one all-reduce of the unfinished count).  A chain of k flat edges ends within
        log2(k) + 1 rounds; what is left after log2(n_flat) + 2 rounds lies on a cycle or leads into one."""
        g, dev, mp = self.part.groups, self.device, self.part.maxpart
        own = g.rank * mp + torch.arange(mp, dtype=torch.int64, device=dev)
        ptr = torch.where(flat, code, own)
        done = ~flat
        for _ in range(n_flat.bit_length() + 2):
            open_ = ~done
            ask = ptr[open_]
            (req,), order, sc, rc = exchange([ask], torch.div(ask, mp, rounding_mode="floor"), g.world)
            loc = req % mp
            ans = torch.stack([ptr[loc], done[loc].to(torch.int64)], 1).reshape(-1)
            back = torch.empty(2 * sum(sc), dtype=torch.int64, device=dev)
            dist.all_to_all_single(back, ans, output_split_sizes=[2 * k for k in sc], input_split_sizes=[2 * k for k in rc])
            got = _unpermute(back.view(-1, 2), order)
            fin = got[:, 1] != 0
            ptr[open_] = torch.where(fin, ask, got[:, 0])
            done[open_] = fin
            left = _global_count(~done)
            if left == 0:
                break
        return torch.tensor(left, dtype=torch.int64, device=dev)

    # ------------------------------------------------------------------------------------------
    # multi-GPU weakly connected components: min-label propagation.  Every owned vertex starts with its own code (owner
    # rank * maxpart + local id, as in bfs / sssp) and is marked changed.  One round: the labels of the changed vertices
    # (INT64_MAX for the others) are all-gathered inside the column group over the block's source slots; the block gives
    # every destination slot the smallest label among its sources (cugraph_b200_block_wcc_min: an atomicMin push over the
    # active columns' edges); ONE MIN reduce-scatter inside the row group brings it to the owner, which keeps it when it is
    # smaller (wcc_owner_step); one all-reduce of the number of changed vertices ends the loop at 0.  The fixpoint is the
    # smallest code of each component: for a given grid it does not depend on timing.
    # ------------------------------------------------------------------------------------------
    def weakly_connected_components(self):
        """Returns (vertices, labels) of the vertices this rank owns: a vertex's label is the external id of one member of
        its component (the same member on every rank), in the vertices' dtype.  The graph must be symmetric (not checked):
        construct it with symmetrize=True, or pass both directions of every edge.  Sets last_wcc_stats = dict(rounds)."""
        p, g = self.part, self.part.groups
        dev, mp = self.device, p.maxpart
        label_own = torch.full((mp,), INT64_MAX, dtype=torch.int64, device=dev)
        label_own[:p.n_local] = g.rank * mp + torch.arange(p.n_local, dtype=torch.int64, device=dev)
        changed = torch.zeros(mp, dtype=torch.bool, device=dev)
        changed[:p.n_local] = True
        label_cols = torch.empty(self.n_cols, dtype=torch.int64, device=dev)
        cand = torch.empty(self.n_rows, dtype=torch.int64, device=dev)
        cand_own = torch.empty(mp, dtype=torch.int64, device=dev)
        rounds = 0
        with _views(label_cols, cand) as (vx, vc):
            while True:
                all_gather_into(label_cols, torch.where(changed, label_own, INT64_MAX), g.col_group)  # the block's column order
                self._call("cugraph_b200_block_wcc_min", self.block, vx.ptr, vc.ptr)
                reduce_scatter_into(cand_own, cand, g.row_group, op=dist.ReduceOp.MIN)
                changed = wcc_owner_step(label_own, cand_own)
                rounds += 1
                if _global_count(changed) == 0:
                    break
        self.last_wcc_stats = dict(rounds=rounds)
        return p.vertices, self._codes_to_external(label_own[:p.n_local])

    # ------------------------------------------------------------------------------------------
    # multi-GPU strongly connected components: single GPU's Multistep (scc.cu) with the owners' state in torch and every
    # round a push over the block (cugraph_b200_block_scc_push); see _SccRun.
    # ------------------------------------------------------------------------------------------
    def strongly_connected_components(self):
        """Returns (vertices, labels) of the vertices this rank owns: a vertex's label is the external id of the member of
        its strongly connected component with the smallest code (owner rank * maxpart + local id), in the vertices' dtype.
        That is the rule of weakly_connected_components, so labels depend on no schedule, every rank agrees on them, and a
        graph that holds every edge in both directions gets weakly_connected_components' labels on the same grid.  Weights
        are ignored, self-loops are never live edges, multi-edges count once per edge.  A graph built with symmetrize=True is
        rejected on every rank (CugraphRuntimeError, single GPU's message).  Sets last_scc_stats = dict(trim_rounds,
        fw_rounds, bw_rounds, outer_rounds, colour_rounds, reach_rounds), the same on every rank."""
        if self.symmetrize:
            raise self._fail("MGGraph.strongly_connected_components",
                             "Invalid input argument: call weakly_connected_components instead for symmetric graphs.")
        run = _SccRun(self)
        try:
            run.trim()
            if run.resolved < self.part.n_global:
                run.forward_backward()
            run.colouring()
            labels = run.labels()
        finally:
            run.close()
        self.last_scc_stats = run.stats
        return self.part.vertices, self._codes_to_external(labels)

    # ------------------------------------------------------------------------------------------
    # multi-GPU Katz, eigenvector centrality and HITS: the single-GPU drivers of centrality.cu with the sweep spread over the
    # grid.  A sweep y = A x over the owners' x is: x all-gathered inside the column group over the block's source slots,
    # the block's pull sweep, ONE reduce-scatter of the partial y inside the row group.  HITS' hub sweep y = A^T x runs the
    # other way round: x all-gathered inside the ROW group over the destination slots (row slot c(v) * maxpart + lid is that
    # group's all-gather order), the block's transposed sweep (cugraph_b200_block_sweep over its column-major copy), ONE
    # reduce-scatter inside the COLUMN group (column slot r(u) * maxpart + lid, the order __init__ already uses for out_w).
    # The owner steps (cugraph_b200_katz_step, ...) pass once over the owned slice and leave fp64 partials on the device;
    # one small all-reduce makes them global, and the one host read per iteration is the convergence test, taken on every
    # rank from the same all-reduced scalars, so that every rank leaves the loop (or raises) in the same iteration.
    # ------------------------------------------------------------------------------------------
    def _spmv(self, x_own, y_own, bufs, alpha, transposed=False, use_weights=True):
        """y_own = alpha * (A x) of the owned vertices (transposed: alpha * (A^T x)); bufs = (x_gathered, y_partial) and
        their views"""
        g = self.part.groups
        xg, yp, vx, vy = bufs
        n_in, in_group = (self.n_rows, g.row_group) if transposed else (self.n_cols, g.col_group)
        n_out, out_group = (self.n_cols, g.col_group) if transposed else (self.n_rows, g.row_group)
        all_gather_into(xg[:n_in], x_own, in_group)
        self._call("cugraph_b200_block_sweep", self.block, 1 if transposed else 0, 1 if use_weights else 0, vx.ptr, vy.ptr,
                   float(alpha))
        reduce_scatter_into(y_own, yp[:n_out], out_group)

    @contextlib.contextmanager
    def _sweep_bufs(self):
        """_spmv's bufs for one orientation, the views freed on exit"""
        xg = torch.zeros(self.x_elems, dtype=self.dtype, device=self.device)    # zero from the span on, as the block sweep requires
        yp = torch.zeros(self.span, dtype=self.dtype, device=self.device)
        with _views(xg, yp) as (vx, vy):
            yield xg, yp, vx, vy

    def _call(self, name, *args):
        """self.lib.<name>(handle, *args, &error), looked up at call time, with its error code checked"""
        err = C.c_void_p()
        code = getattr(self.lib, name)(self.handle.ptr, *args, C.byref(err))
        self._capi.check(code, err, name)

    @staticmethod
    def _fail(where, message):
        """the error the single-GPU entry point returns (CUGRAPH_UNKNOWN_ERROR -> RuntimeError), with its message"""
        from cugraph_b200 import _capi as capi
        return capi.CugraphRuntimeError(capi.UNKNOWN_ERROR, message, where)

    def katz_centrality(self, alpha, beta=1.0, epsilon=1e-6, max_iterations=100):
        """Katz centrality (cugraph_katz_centrality's semantics): x <- alpha * A^T x + beta from x = 0 until
        sum |x_new - x| < epsilon (compared in the block's dtype), then x / ||x||_2.  Edge weights are used.
        Returns (vertices, values) of the vertices this rank owns; sets last_katz_stats = dict(iterations)."""
        from cugraph_b200 import _capi as capi
        p, dev, dt, mp = self.part, self.device, self.dtype, self.part.maxpart
        if not 0.0 <= alpha <= 1.0:
            raise capi.CugraphValueError(capi.INVALID_INPUT, "Invalid input argument: alpha should be in [0.0, 1.0].",
                                         "MGGraph.katz_centrality")
        if not epsilon >= 0.0:
            raise capi.CugraphValueError(capi.INVALID_INPUT, "Invalid input argument: epsilon should be non-negative.",
                                         "MGGraph.katz_centrality")
        T = _np_type(dt)
        x = torch.zeros(mp, dtype=dt, device=dev)
        y = torch.zeros(mp, dtype=dt, device=dev)
        part = torch.zeros(2, dtype=torch.float64, device=dev)
        it = 0
        with self._sweep_bufs() as bufs, _views(x, y) as (vxo, vyo):
            while True:
                self._spmv(x, y, bufs, alpha)
                part.zero_()
                self._call("cugraph_b200_katz_step", vyo.ptr, vxo.ptr, p.n_local, float(beta), C.c_void_p(part.data_ptr()))
                dist.all_reduce(part)
                diff, sumsq = part.tolist()
                it += 1
                if T(diff) < T(epsilon):
                    break
                if it >= max_iterations:
                    raise self._fail("MGGraph.katz_centrality", "Katz Centrality failed to converge.")
            l2 = math.sqrt(sumsq)           # the last step's sum of x_new^2 = ||x||^2
            if not l2 > 0.0:
                raise self._fail("MGGraph.katz_centrality", "L2 norm of the computed Katz Centrality values should be positive.")
            self._call("cugraph_b200_vertex_scale", vxo.ptr, p.n_local, 1.0 / l2)
        self.last_katz_stats = dict(iterations=it)
        return p.vertices, x[:p.n_local].clone()

    def eigenvector_centrality(self, epsilon=1e-6, max_iterations=100):
        """Eigenvector centrality (cugraph_eigenvector_centrality's semantics): x <- (A^T x + x) / ||A^T x + x||_2 from
        x = 1 / V until sum |x_new - x| < V * epsilon (V = the global vertex count, compared in the block's dtype).  Edge
        weights are used.  Returns (vertices, values) of the vertices this rank owns; sets last_eigenvector_stats."""
        from cugraph_b200 import _capi as capi
        p, dev, dt, mp = self.part, self.device, self.dtype, self.part.maxpart
        if not epsilon >= 0.0:
            raise capi.CugraphValueError(capi.INVALID_INPUT, "Invalid input argument: epsilon should be non-negative.",
                                         "MGGraph.eigenvector_centrality")
        T = _np_type(dt)
        V = p.n_global
        x = torch.zeros(mp, dtype=dt, device=dev)
        x[:p.n_local] = 1.0 / V
        y = torch.zeros(mp, dtype=dt, device=dev)
        sq = torch.zeros(1, dtype=torch.float64, device=dev)
        part = torch.zeros(1, dtype=torch.float64, device=dev)
        tolerance = T(V) * T(epsilon)
        it = 0
        with self._sweep_bufs() as bufs, _views(x, y) as (vxo, vyo):
            while True:
                self._spmv(x, y, bufs, 1.0)
                sq.zero_()
                self._call("cugraph_b200_eigenvector_add_step", vyo.ptr, vxo.ptr, p.n_local, C.c_void_p(sq.data_ptr()))
                dist.all_reduce(sq)
                part.zero_()
                self._call("cugraph_b200_eigenvector_scale_step", vyo.ptr, vxo.ptr, p.n_local, C.c_void_p(sq.data_ptr()),
                           C.c_void_p(part.data_ptr()))
                dist.all_reduce(part)
                diff = float(part.item())
                it += 1
                if T(diff) < tolerance:
                    break
                if it >= max_iterations:
                    raise self._fail("MGGraph.eigenvector_centrality", "Eigenvector Centrality failed to converge.")
        self.last_eigenvector_stats = dict(iterations=it)
        return p.vertices, x[:p.n_local].clone()

    def _owned_lids(self, ids):
        """(local ids, hit) of int64 external ids sent to this rank as their owner: hit[i] says whether ids[i] is a vertex
        of the graph, and then lid[i] is its local id (lid[i] is 0 where it is not)"""
        p, n = self.part, self.part.n_local
        if n == 0 or ids.numel() == 0:
            return (torch.zeros(ids.numel(), dtype=torch.int64, device=ids.device),
                    torch.zeros(ids.numel(), dtype=torch.bool, device=ids.device))
        if self._id_order is None:   # sorted once per graph: a sort of the owned ids costs milliseconds at scale
            vid = p.vertices.to(torch.int64)
            order = torch.argsort(vid)
            self._id_order = (order, vid[order])
        order, sv = self._id_order
        pos = torch.searchsorted(sv, ids).clamp(max=n - 1)
        hit = sv[pos] == ids
        return torch.where(hit, order[pos], 0), hit

    def _pairs_to_owners(self, pairs, dtype):
        """(vertex ids, values) given by this rank (None: nothing) for any vertices -> the pairs of the vertices this rank
        owns, from every rank, with one all-to-all-v (every rank must call it).  Returns (local ids, values in `dtype`,
        counts): the received pairs whose id is a vertex of the graph, and this rank's float64 counts [ids and values differ
        in size (then nothing is sent), pairs sent, negative values sent, ids received that are not vertices, ids received
        more than once] for the caller's one all-reduce."""
        p, g, dev = self.part, self.part.groups, self.device
        gv = torch.zeros(0, dtype=torch.int64, device=dev)
        gx = torch.zeros(0, dtype=dtype, device=dev)
        mismatch = 0
        if pairs is not None:
            v = torch.as_tensor(pairs[0]).to(dev).to(torch.int64).reshape(-1)
            x = torch.as_tensor(pairs[1]).to(dev).to(dtype).reshape(-1)
            if v.numel() == x.numel():
                gv, gx = v, x
            else:
                mismatch = 1
        (rv, rx), _, _, _ = exchange([gv, gx], vertex_owner(gv, g.world), g.world)
        lid, hit = self._owned_lids(rv)
        lid, val = lid[hit], rx[hit]
        srt = torch.sort(lid).values
        counts = torch.stack([torch.tensor(mismatch, dtype=torch.float64, device=dev),
                              torch.tensor(gv.numel(), dtype=torch.float64, device=dev),
                              (gx < 0).sum().to(torch.float64), (~hit).sum().to(torch.float64),
                              (srt[1:] == srt[:-1]).sum().to(torch.float64)])
        return lid, val, counts

    def hits(self, epsilon=1e-5, max_iterations=100, initial_hubs_guess=None, normalize=True):
        """HITS (cugraph_hits' semantics): authorities = A^T hubs, hubs = A authorities (the hubs sweep reads the authorities
        before their normalisation), both divided by their maximum, until sum |hubs - previous hubs| < V * epsilon (V = the
        global vertex count, compared in the block's dtype); then both divided by their sum when `normalize`.  Edge weights
        are not used.  initial_hubs_guess = (vertex ids, values), from any rank for any vertices (others start at 0),
        L1-normalised.  Returns (vertices, hubs, authorities) of the vertices this rank owns; sets
        last_hits_stats = dict(iterations, hub_score_differences)."""
        from cugraph_b200 import _capi as capi
        p, dev, dt, mp = self.part, self.device, self.dtype, self.part.maxpart
        if not epsilon >= 0.0:
            raise capi.CugraphValueError(capi.INVALID_INPUT, "Invalid input argument: epsilon should be non-negative.",
                                         "MGGraph.hits")
        T = _np_type(dt)
        V = p.n_global
        prev = torch.zeros(mp, dtype=dt, device=dev)
        curr = torch.zeros(mp, dtype=dt, device=dev)
        auth = torch.zeros(mp, dtype=dt, device=dev)
        mx = torch.zeros(2, dtype=torch.float64, device=dev)
        part = torch.zeros(2, dtype=torch.float64, device=dev)
        where = "MGGraph.hits"

        def l1_normalize(views):
            part.zero_()
            for k, v in enumerate(views):
                self._call("cugraph_b200_vertex_sum", v.ptr, p.n_local, 0, C.c_void_p(part.data_ptr() + 8 * k))
            dist.all_reduce(part)
            norms = part.tolist()
            for k, v in enumerate(views):
                if not T(norms[k]) > T(0):
                    raise self._fail(where, "Norm is required to be a positive value.")
                self._call("cugraph_b200_vertex_scale", v.ptr, p.n_local, 1.0 / norms[k])

        with self._sweep_bufs() as pull_bufs, self._sweep_bufs() as push_bufs, _views(prev, curr, auth) as (vp, vc, va):
            has = torch.tensor([0 if initial_hubs_guess is None else 1], dtype=torch.int64, device=dev)
            dist.all_reduce(has, op=dist.ReduceOp.MAX)   # a guess from any rank: every rank takes part in its exchange
            if int(has.item()):
                lid, val, counts = self._pairs_to_owners(initial_hubs_guess, dt)
                dist.all_reduce(counts)
                mismatch, _, neg, _, _ = counts.tolist()
                if mismatch:
                    raise capi.CugraphValueError(capi.INVALID_INPUT,
                                                 "initial hubs guess needs vertices and values of equal size", where)
                if neg:
                    raise capi.CugraphValueError(capi.INVALID_INPUT,
                                                 "Invalid input argument: initial guess values should be non-negative.", where)
                prev[lid] = val                              # ids that are not vertices of the graph are dropped
                l1_normalize([vp])
            else:
                prev[:p.n_local] = 1.0 / V
            tolerance = T(V) * T(epsilon)
            it, diff = 0, float(np.finfo(T).max)
            while True:
                self._spmv(prev, auth, pull_bufs, 1.0, use_weights=False)
                self._spmv(auth, curr, push_bufs, 1.0, transposed=True, use_weights=False)
                mx.zero_()
                self._call("cugraph_b200_hits_max_step", vc.ptr, va.ptr, p.n_local, C.c_void_p(mx.data_ptr()))
                dist.all_reduce(mx, op=dist.ReduceOp.MAX)
                part.zero_()
                self._call("cugraph_b200_hits_scale_step", vc.ptr, va.ptr, vp.ptr, p.n_local, C.c_void_p(mx.data_ptr()),
                           C.c_void_p(part.data_ptr()))
                dist.all_reduce(part)
                d, h_max, a_max = torch.cat([part[:1], mx]).tolist()
                if not (T(h_max) > T(0) and T(a_max) > T(0)):
                    raise self._fail(where, "Norm is required to be a positive value.")
                diff = float(T(d))
                prev, curr, vp, vc = curr, prev, vc, vp
                it += 1
                if T(diff) < tolerance:
                    break
                if it >= max_iterations:
                    raise self._fail(where, "HITS failed to converge.")
            if normalize:
                l1_normalize([vp, va])
        self.last_hits_stats = dict(iterations=it, hub_score_differences=diff)
        return p.vertices, prev[:p.n_local].clone(), auth[:p.n_local].clone()


def _unpermute(x, order):
    """the answers of an exchange() in the order of the requests: x[k] answers request order[k]"""
    out = torch.empty_like(x)
    out[order] = x
    return out


def _is_scalar(x):
    """a Python / NumPy integer or a 0-d tensor / array: MGGraph.bfs's one-source form"""
    if isinstance(x, (torch.Tensor, np.ndarray)):
        return x.ndim == 0
    return isinstance(x, (int, np.integer))


def _np_type(dtype):
    """the numpy scalar type of a block dtype: convergence tests compare in it, as the single-GPU drivers compare in T"""
    return np.float32 if dtype == torch.float32 else np.float64


INT64_MAX = torch.iinfo(torch.int64).max


def window_bound(lo, delta, dtype, device):
    """upper bound lo + delta of a Δ-window as a 0-d tensor of the distance dtype, strictly above lo after rounding"""
    lo_t = torch.tensor(lo, dtype=dtype)
    hi_t = torch.tensor(lo + delta, dtype=dtype)
    if not bool(hi_t > lo_t):
        hi_t = torch.nextafter(lo_t, torch.tensor(math.inf, dtype=dtype))
    return hi_t.to(device)


def sssp_owner_step(dist_own, pred_code, pending, cand_own):
    """The owner's step of one multi-GPU SSSP round: decode the reduced keys (cugraph_b200_block_sssp_relax; INT64_MAX = no
    proposal), accept strict improvements of dist_own, mark them pending and, for float keys, take the predecessor code from
    the key's low 32 bits.  Updates the arrays in place and returns the mask of improved vertices."""
    if dist_own.dtype == torch.float32:
        d = (cand_own >> 32).to(torch.int32).view(torch.float32)
    else:
        d = cand_own.view(torch.float64)
    improved = (cand_own != INT64_MAX) & (d < dist_own)
    dist_own.copy_(torch.where(improved, d, dist_own))
    pending |= improved
    if dist_own.dtype == torch.float32:
        pred_code.copy_(torch.where(improved, cand_own & 0xFFFFFFFF, pred_code))
    return improved


def wcc_owner_step(label_own, cand_own):
    """The owner's step of one multi-GPU WCC round: keep the reduced candidate label (cugraph_b200_block_wcc_min; INT64_MAX =
    no active neighbour) where it is smaller than label_own.  Updates label_own in place and returns the mask of changed
    vertices."""
    changed = cand_own < label_own
    label_own.copy_(torch.where(changed, cand_own, label_own))
    return changed


INT64_MIN = torch.iinfo(torch.int64).min
SCC_PUSH_MAX, SCC_PUSH_COUNT = 0, 1   # the modes of cugraph_b200_block_scc_push


class _SccRun:
    """One call of MGGraph.strongly_connected_components: single GPU's Multistep (scc.cu), phase by phase.

    Owner state over the maxpart slots (int64 or bool; padding slots are never live): `live`, `sub` (subproblem of a live
    vertex, -1 otherwise), `comp` (a member code of a resolved vertex's SCC), the live in- and out-degree counts and the
    colour.  One round: the active sources' values (INT64_MIN = inactive) are all-gathered over the block's source slots
    (forward: column slots, in the column group; backward: row slots, in the row group); cugraph_b200_block_scc_push pushes
    them over the edges whose source and destination keys agree; ONE reduce-scatter (MAX or SUM) brings the result to the
    destinations' owners (forward: row group; backward: column group); a torch owner step; one all-reduce of the number of
    changed vertices ends the loop on every rank at once.  The keys (subproblem or colour, over the source and the
    destination slots) change only between phases and colouring rounds and are gathered then.
      1. trim: live in- / out-degrees by a count push in both orientations; vertices with a zero count are peeled, and their
         edges, pushed in both orientations as counts, are the next round's decrements.  Vertices without edges are peeled
         at once: singletons.
      2. forward-backward from the live vertex with the largest in-degree x out-degree, ties to the smallest code (two
         all-reduces): FW and BW reach inside the pivot's subproblem; FW ∩ BW is resolved, FW\\BW, BW\\FW and the rest
         become subproblems 1, 2 and 3.
      3. colouring until nothing is live: the largest code flows forward inside a subproblem (max push), the roots (colour
         = own code) reach backward among the vertices of their colour, the reached vertices are resolved, every other live
         vertex takes its colour as its subproblem.  An outer round that resolves nothing raises on every rank.
    Labels: the smallest member code of every SCC, by one all-to-all-v of (comp, code) to comp's owner and one back."""

    def __init__(self, graph):
        self.G = graph
        p, g = graph.part, graph.part.groups
        self.p, self.g, self.mp = p, g, p.maxpart
        dev, mp, i64 = graph.device, p.maxpart, torch.int64
        self.code = torch.full((mp,), -1, dtype=i64, device=dev)
        self.code[:p.n_local] = g.rank * mp + torch.arange(p.n_local, dtype=i64, device=dev)
        self.live = self.code >= 0
        self.sub = torch.full((mp,), -1, dtype=i64, device=dev)
        self.comp = self.code.clone()
        self.deg_in = torch.empty(mp, dtype=i64, device=dev)
        self.deg_out = torch.empty(mp, dtype=i64, device=dev)
        self.got = torch.empty(mp, dtype=i64, device=dev)
        self.got2 = torch.empty(mp, dtype=i64, device=dev)
        nc, nr = graph.n_cols, graph.n_rows
        self.key_c, self.val_c, self.out_c = (torch.zeros(nc, dtype=i64, device=dev) for _ in range(3))
        self.key_r, self.val_r, self.out_r = (torch.zeros(nr, dtype=i64, device=dev) for _ in range(3))
        self._views = _views(self.key_c, self.val_c, self.out_c, self.key_r, self.val_r, self.out_r)
        self.vkc, self.vvc, self.voc, self.vkr, self.vvr, self.vor = self._views.__enter__()
        self.resolved = 0
        self.stats = dict(trim_rounds=0, fw_rounds=0, bw_rounds=0, outer_rounds=0, colour_rounds=0, reach_rounds=0)

    def close(self):
        self._views.__exit__(None, None, None)

    def push(self, backward, mode, val_own, out_own):
        """out_own = the owners' reduced push of val_own (INT64_MIN = inactive source) along the edges, or against them"""
        G, g = self.G, self.g
        op = dist.ReduceOp.MAX if mode == SCC_PUSH_MAX else dist.ReduceOp.SUM
        if backward:
            all_gather_into(self.val_r, val_own, g.row_group)
            G._call("cugraph_b200_block_scc_push", G.block, 1, mode, self.vkr.ptr, self.vvr.ptr, self.vkc.ptr, self.mp, g.R,
                    g.C, g.r, g.c, self.voc.ptr)
            reduce_scatter_into(out_own, self.out_c, g.col_group, op=op)
        else:
            all_gather_into(self.val_c, val_own, g.col_group)
            G._call("cugraph_b200_block_scc_push", G.block, 0, mode, self.vkc.ptr, self.vvc.ptr, self.vkr.ptr, self.mp, g.R,
                    g.C, g.r, g.c, self.vor.ptr)
            reduce_scatter_into(out_own, self.out_r, g.row_group, op=op)
        return out_own

    def gather_keys(self, key_own):
        all_gather_into(self.key_c, key_own, self.g.col_group)
        all_gather_into(self.key_r, key_own, self.g.row_group)

    def resolve(self, done, member):
        """done (a mask of live vertices) is resolved with comp = member; returns the global count (one all-reduce)"""
        self.comp = torch.where(done, member, self.comp)
        self.live &= ~done
        self.sub = torch.where(self.live, self.sub, -1)
        n = _global_count(done)
        self.resolved += n
        return n

    def trim(self):
        self.key_c.zero_()
        self.key_r.zero_()
        self.push(False, SCC_PUSH_COUNT, torch.where(self.live, 0, INT64_MIN), self.deg_in)
        self.push(True, SCC_PUSH_COUNT, torch.where(self.live, 0, INT64_MIN), self.deg_out)
        self.sub = torch.where(self.live, 0, -1)
        rounds = 0
        peel = self.live & ((self.deg_in == 0) | (self.deg_out == 0))
        while self.resolve(peel, self.code):
            val = torch.where(peel, 0, INT64_MIN)
            self.deg_in -= self.push(False, SCC_PUSH_COUNT, val, self.got)
            self.deg_out -= self.push(True, SCC_PUSH_COUNT, val, self.got2)
            peel = self.live & ((self.deg_in == 0) | (self.deg_out == 0))
            rounds += 1
        self.stats["trim_rounds"] = rounds

    def reach(self, backward, mark):
        """mark |= the vertices reached from mark (along the edges, or against them) with the source's key; returns the
        rounds"""
        frontier, rounds = mark, 0
        while True:
            got = self.push(backward, SCC_PUSH_MAX, torch.where(frontier, 0, INT64_MIN), self.got)
            frontier = self.live & ~mark & (got != INT64_MIN)
            mark |= frontier
            rounds += 1
            if _global_count(frontier) == 0:
                return rounds

    def forward_backward(self):
        score = torch.where(self.live, self.deg_in * self.deg_out, -1).max().reshape(1)
        dist.all_reduce(score, op=dist.ReduceOp.MAX)
        pivot = torch.where(self.live & (self.deg_in * self.deg_out == score), self.code, INT64_MAX).min().reshape(1)
        dist.all_reduce(pivot, op=dist.ReduceOp.MIN)
        self.gather_keys(self.sub)
        fw, bw = self.code == pivot, self.code == pivot
        self.stats["fw_rounds"] = self.reach(False, fw)
        self.stats["bw_rounds"] = self.reach(True, bw)
        self.sub = torch.where(fw, 1, torch.where(bw, 2, 3))
        self.resolve(self.live & fw & bw, pivot)

    def colouring(self):
        st = self.stats
        while self.resolved < self.p.n_global:
            self.gather_keys(self.sub)
            colour = torch.where(self.live, self.code, -1)
            frontier = self.live
            while True:
                got = self.push(False, SCC_PUSH_MAX, torch.where(frontier, colour, INT64_MIN), self.got)
                frontier = self.live & (got > colour)
                colour = torch.where(frontier, got, colour)
                st["colour_rounds"] += 1
                if _global_count(frontier) == 0:
                    break
            self.gather_keys(colour)
            roots = self.live & (colour == self.code)
            st["reach_rounds"] += self.reach(True, roots)
            self.sub = colour
            if self.resolve(roots, colour) == 0:
                raise MGGraph._fail("MGGraph.strongly_connected_components",
                                    "strongly_connected_components: a colouring round resolved no vertex")
            st["outer_rounds"] += 1

    def labels(self):
        """the smallest member code of every owned vertex's SCC"""
        p, g, mp = self.p, self.g, self.mp
        comp, code = self.comp[:p.n_local], self.code[:p.n_local]
        (lid, member), order, sc, rc = exchange([comp % mp, code], torch.div(comp, mp, rounding_mode="floor"), g.world)
        low = torch.full((mp,), INT64_MAX, dtype=torch.int64, device=comp.device).scatter_reduce_(0, lid, member, "amin")
        back = torch.empty(sum(sc), dtype=torch.int64, device=comp.device)
        dist.all_to_all_single(back, low[lid].contiguous(), output_split_sizes=sc, input_split_sizes=rc)
        label = torch.empty_like(back)
        label[order] = back
        return label


def bfs(graph: MGGraph, sources, depth_limit=-1, compute_predecessors=True, *, direction_optimizing=False):
    """(vertices, distances, predecessors) of the vertices owned by this rank (the MG contract of pylibcugraph.bfs).
    sources: one external id, the same on every rank, or a 1-D tensor / array of this rank's source ids;
    direction_optimizing: top-down on every level (False) or single GPU's per-level switch (True) (see MGGraph.bfs)."""
    return graph.bfs(sources, depth_limit, compute_predecessors, direction_optimizing=direction_optimizing)


def multi_source_bfs(graph: MGGraph, sources, depth_limit=-1, compute_predecessors=True, *, direction_optimizing=False):
    """(vertices, distances [n, n_local], predecessors [n, n_local]) of the vertices owned by this rank: one BFS per source,
    row k from sources[k]; sources is the same list on every rank (see MGGraph.multi_source_bfs)."""
    return graph.multi_source_bfs(sources, depth_limit, compute_predecessors, direction_optimizing=direction_optimizing)


def validate_bfs(graph: MGGraph, vertices, distances, predecessors, sources, depth_limit=-1):
    """the certificate of a BFS result given as this rank's (vertices, distances, predecessors): a dict, the same on every
    rank (see MGGraph.validate_bfs)"""
    return graph.validate_bfs(vertices, distances, predecessors, sources, depth_limit)


def validate_sssp(graph: MGGraph, vertices, distances, predecessors, source, cutoff=math.inf):
    """the certificate of an SSSP result given as this rank's (vertices, distances, predecessors): a dict, the same on
    every rank (see MGGraph.validate_sssp)"""
    return graph.validate_sssp(vertices, distances, predecessors, source, cutoff)


def rmat_edgelist_share(scale, num_edges, a=0.57, b=0.19, c=0.19, seed=0, clip_and_flip=False, scramble_ids=True,
                        groups: Groups | None = None, device="cuda"):
    """This rank's slice [r * E // P, (r + 1) * E // P) of the global RMAT stream of `seed` (E = num_edges, P ranks, r this
    rank), generated on its own: returns (src, dst, first), first = the slice's first edge index.  The stream is counter-based
    (cugraph_b200_generate_rmat_edgelist_at), so the ranks' slices in rank order are the single-call output
    generators.rmat_edgelist(scale, E, ...) bit for bit, whatever P is; values drawn per edge at the same global indices
    (generators.uniform_values(..., first=first)) stay attached to the same edges.  groups: the grid's Groups (default:
    the default process group)."""
    from cugraph_b200.generators import rmat_edgelist
    rank, world = (groups.rank, groups.world) if groups is not None else (dist.get_rank(), dist.get_world_size())
    first = rank * int(num_edges) // world
    count = (rank + 1) * int(num_edges) // world - first
    src, dst = rmat_edgelist(scale, count, a, b, c, seed, scramble_ids, clip_and_flip, device=device, first_edge=first)
    return src, dst, first


def extract_paths(graph: MGGraph, distances, predecessors, destinations):
    """(paths, max_path_length) for this rank's destinations from this rank's part of a BFS result (the MG contract of
    pylibcugraph.extract_paths; see MGGraph.extract_paths)."""
    return graph.extract_paths(distances, predecessors, destinations)


def sssp(graph: MGGraph, source, cutoff=math.inf, compute_predecessors=True):
    """(vertices, distances, predecessors) of the vertices owned by this rank (the MG contract of pylibcugraph.sssp;
    predecessors are None when not requested)."""
    return graph.sssp(source, cutoff, compute_predecessors)


def weakly_connected_components(graph: MGGraph):
    """(vertices, labels) of the vertices owned by this rank (the MG contract of pylibcugraph.weakly_connected_components;
    the graph must be symmetric: MGGraph(..., symmetrize=True))."""
    return graph.weakly_connected_components()


def strongly_connected_components(graph: MGGraph):
    """(vertices, labels) of the vertices owned by this rank (the MG contract of pylibcugraph.strongly_connected_components;
    see MGGraph.strongly_connected_components)."""
    return graph.strongly_connected_components()


def degrees(graph: MGGraph):
    """(vertices, in_degrees, out_degrees) of the vertices owned by this rank (the MG contract of pylibcugraph.degrees)."""
    return graph.degrees()


def katz_centrality(graph: MGGraph, alpha, beta=1.0, epsilon=1e-6, max_iterations=100):
    """(vertices, values) of the vertices owned by this rank (the MG contract of pylibcugraph.katz_centrality)."""
    return graph.katz_centrality(alpha, beta, epsilon, max_iterations)


def eigenvector_centrality(graph: MGGraph, epsilon=1e-6, max_iterations=100):
    """(vertices, values) of the vertices owned by this rank (the MG contract of pylibcugraph.eigenvector_centrality)."""
    return graph.eigenvector_centrality(epsilon, max_iterations)


def hits(graph: MGGraph, epsilon=1e-5, max_iterations=100, initial_hubs_guess=None, normalize=True):
    """(vertices, hubs, authorities) of the vertices owned by this rank (the MG contract of pylibcugraph.hits)."""
    return graph.hits(epsilon, max_iterations, initial_hubs_guess, normalize)


def pagerank(graph: MGGraph, alpha=0.85, epsilon=1e-5, max_iterations=100, *, initial_guess=None,
             precomputed_out_weights=None, fail_on_nonconvergence=False):
    """Returns (vertices, pageranks, converged) for the vertices owned by this rank
    (the MG contract of pylibcugraph.pagerank: every rank gets its local part).  The keywords are MGGraph.pagerank's."""
    v, p, it, conv = graph.pagerank(alpha, epsilon, max_iterations, initial_guess=initial_guess,
                                    precomputed_out_weights=precomputed_out_weights,
                                    fail_on_nonconvergence=fail_on_nonconvergence)
    return v, p, conv


def personalized_pagerank(graph: MGGraph, personalization, alpha=0.85, epsilon=1e-5, max_iterations=100, *,
                          initial_guess=None, precomputed_out_weights=None, fail_on_nonconvergence=False):
    """Returns (vertices, pageranks, converged) for the vertices owned by this rank (the MG contract of
    pylibcugraph.personalized_pagerank).  personalization = (external vertex ids, values) from this rank, or None when
    another rank gives them; the keywords are MGGraph.pagerank's."""
    v, p, it, conv = graph.pagerank(alpha, epsilon, max_iterations, personalization=personalization,
                                    initial_guess=initial_guess, precomputed_out_weights=precomputed_out_weights,
                                    fail_on_nonconvergence=fail_on_nonconvergence)
    return v, p, conv
