"""Multi-GPU BFS top-down and direction-optimising (MGGraph.bfs(direction_optimizing=...)) on every rank of a grid in ONE
process (tests/mg_world.py), the graphs, the schedules and the checks, with numpy restatements of the two new entry
points: cugraph_b200_block_bfs_push on one block and Beamer's rule behind cugraph_b200_bfs_bottom_up.

Shared by tests/test_mg_bfs_direction_cpu.py and tests/test_mg_bfs_direction_gpu.py."""
import ctypes as C
import re

import numpy as np

import oracle
from tests import mg_paths_ref as refs
from tests import mg_world
from tests import test_traversal_shapes_gpu as shapes

# name -> (direction_optimizing, knobs).  "bottom_up" is the schedule of the pull-only driver: every level whose frontier
# has out-edges runs bottom-up; "flip" switches to bottom-up on the first level and back whenever the frontier shrinks.
SCHEDULES = {
    "top_down": (False, {}),
    "optimizing": (True, {}),
    "bottom_up": (True, {"CUGRAPH_B200_BFS_ALPHA": "1e30", "CUGRAPH_B200_BFS_BETA": "1e30"}),
    "flip": (True, {"CUGRAPH_B200_BFS_ALPHA": "1e6", "CUGRAPH_B200_BFS_BETA": "1e-6"}),
}
KNOBS = ("CUGRAPH_B200_BFS_ALPHA", "CUGRAPH_B200_BFS_BETA")


def set_knobs(monkeypatch, knobs):
    """the schedule's knobs in the environment (read when a handle is created), the others unset"""
    for k in KNOBS:
        if k in knobs:
            monkeypatch.setenv(k, knobs[k])
        else:
            monkeypatch.delenv(k, raising=False)


# ---------------------------------------------------------------------------------------------------- graphs
class Case:
    """a directed edge list over vertex indices (s, d), the external id of every index (ids: None = the index itself),
    per-rank source lists (indices) by world size, and whether the edge list is symmetric"""

    def __init__(self, name, s, d, sources, ids=None, symmetric=False):
        self.name, self.s, self.d, self.ids, self.symmetric = name, np.asarray(s, np.int32), np.asarray(d, np.int32), ids, symmetric
        self.sources = np.asarray(sources, np.int32)    # the union of every rank's sources

    def per_rank(self, world, rng):
        return refs.split(self.sources, world, rng)


def _sym(s, d):
    return np.concatenate([s, d]), np.concatenate([d, s])


def _with_out_edges(s, k, rng):
    return rng.choice(np.flatnonzero(np.bincount(s) > 0), k, replace=False).astype(np.int32)


def cases(sz, scale):
    """the graphs: directed and symmetrised RMAT, a path with random ids (int64 external ids), a grid with edges removed,
    a lollipop, a union of small components (many sources) and the forest with forced predecessors"""
    rng = np.random.default_rng(scale)
    out = []
    s, d = refs.rmat_graph(scale)
    out.append(Case("rmat-directed", s, d, _with_out_edges(s, 3, rng)))
    s2, d2 = _sym(s, d)
    out.append(Case("rmat-symmetric", s2, d2, _with_out_edges(s2, 1, rng), symmetric=True))
    p = shapes.path(sz["path"], "random")
    ids64 = (10**12 + 7 * p.ids.astype(np.int64))
    ps, pd = _sym(p.s, p.d)
    out.append(Case("path-int64-ids", ps, pd, [sz["path"] // 3], ids=ids64, symmetric=True))
    gr = shapes.grid(sz["grid"])
    out.append(Case("grid", gr.s, gr.d, gr.source_sets[0]))
    lo = shapes.lollipop(sz["core"], sz["tail"], sz["clique"])
    ls, ld = _sym(lo.s, lo.d)
    out.append(Case("lollipop", ls, ld, lo.source_sets[0], symmetric=True))
    co = shapes.components(sz["components"])
    cs, cd = _sym(co.s, co.d)
    out.append(Case("components", cs, cd, co.source_sets[0], symmetric=True))
    fs, fd, roots, _ = refs.forced_graph()
    out.append(Case("forced", fs, fd, roots))
    return out


# ---------------------------------------------------------------------------------------------------- the runs
def _worker(rank, world, case, sources, do, limits, dests, device):
    import torch

    def ext(a):   # indices -> external ids; an index past the vertices -> a small id that is not a vertex either
        if case.ids is None:
            return a
        a = np.asarray(a, np.int64)
        return np.where(a < case.ids.size, case.ids[np.minimum(a, case.ids.size - 1)], 5 + a)

    g = mg_world.graph(rank, world, ext(case.s), ext(case.d), device=device)
    order = None if case.ids is None else np.argsort(case.ids)

    def index(x):   # external ids -> indices (-1 stays -1)
        x = x.cpu().numpy().astype(np.int64)
        if order is None:
            return x
        pos = np.searchsorted(case.ids[order], np.where(x >= 0, x, case.ids.min())).clip(max=order.size - 1)
        return np.where(x >= 0, order[pos], -1)

    src = torch.as_tensor(ext(sources[rank])).to(device)
    runs = []
    for limit in limits:
        v, dist, pred = g.bfs(src, limit, direction_optimizing=do)
        r = dict(v=index(v), dist=dist.cpu().numpy(), pred=index(pred), n_local=g.part.n_local, limit=limit,
                 stats=dict(g.last_bfs_stats))
        if limit < 0:
            again = g.bfs(src, limit, direction_optimizing=do)[2]
            r["pred_again"] = index(again)
            paths, length = g.extract_paths(dist, pred, torch.as_tensor(ext(dests[rank])).to(device))
            r.update(paths=index(paths.reshape(-1)).reshape(paths.shape), length=length,
                     rounds=g.last_paths_stats["rounds"])
        runs.append(r)
    return runs


def depth(case):
    """D: the largest finite BFS distance from the case's sources"""
    ids, remap = mg_world.present(case.s, case.d, int(max(case.s.max(), case.d.max())) + 1)
    ref_d, _ = oracle.bfs(remap[case.s].astype(np.int32), remap[case.d].astype(np.int32), ids.size,
                          remap[np.unique(case.sources)].astype(np.int32))
    ref_d = np.asarray(ref_d, np.int64)
    return int(ref_d[(ref_d >= 0) & (ref_d < refs.IMAX)].max())


def run_case(case, world, schedule, rng, device="cpu", limits=True):
    """MGGraph.bfs on `world` ranks (the grid and knobs set by the caller) from the case's sources dealt to the ranks:
    unlimited, then with depth limits 1, D / 2, D and D + 1; every check of the module.  Returns the unlimited run's
    per-rank dicts."""
    do, _ = SCHEDULES[schedule]
    D = depth(case)
    lims = [-1] + ([1, max(D // 2, 1), D, D + 1] if limits else [])
    ids = np.unique(np.concatenate([case.s, case.d]))
    pool = np.concatenate([rng.choice(ids, 40), case.sources, refs.not_vertices(case.s, case.d, 2)]).astype(np.int32)
    dests = refs.split(pool, world, rng)
    out = mg_world.run(world, _worker, case, case.per_rank(world, rng), do, lims, dests, device)
    for k, limit in enumerate(lims):
        res = [r[k] for r in out]
        what = f"{case.name} {schedule} depth_limit={limit}"
        stats = res[0]["stats"]
        assert all(r["stats"] == stats for r in res), what
        assert stats["levels"] == stats["top_down"] + stats["bottom_up"], what
        if not do:
            assert stats["bottom_up"] == 0, what
        if schedule == "bottom_up":
            assert stats["top_down"] == 0, what
        got_d = refs.check_bfs(case.s, case.d, res, case.sources, depth_limit=limit)
        if limit < 0:
            assert got_d[got_d < refs.IMAX].max() == D, what
            assert stats["levels"] == D + 1, what
            for r in res:
                assert np.array_equal(r["pred_again"], r["pred"]), what
            refs.check_paths(res, dests)
        else:
            assert stats["levels"] == min(limit, D + 1), what
    return [r[0] for r in out]


# ---------------------------------------------------------------------------------------------------- single GPU
def single_gpu_bfs(s, d, sources, direction_optimizing, symmetric):
    """cugraph_bfs on the single-GPU graph of the edges: (distances, predecessors) by vertex id, -5 for non-vertices"""
    from tests.gpu_util import make_graph
    from tests.test_paths_gpu import _bfs
    h, g = make_graph(s, d, symmetric=symmetric)
    verts, dist, pred = _bfs(h, g, sources, direction_optimizing)
    v = verts.cpu().numpy()
    n = int(max(s.max(), d.max())) + 1
    out_d, out_p = np.full(n, -5, np.int64), np.full(n, -5, np.int64)
    out_d[v] = dist.cpu().numpy()
    out_p[v] = pred.cpu().numpy()
    return out_d, out_p


def trace_directions(text):
    """(top-down, bottom-up) level counts of a CUGRAPH_B200_BFS_TRACE log"""
    dirs = re.findall(r"^bfs level \d+ (top-down|bottom-up) ", text, flags=re.M)
    return dirs.count("top-down"), dirs.count("bottom-up")


# ---------------------------------------------------------------------------------------------------- entry points
def code_of(col, maxpart, grid_cols, grid_c):
    """column_code: owner rank * maxpart + local id of a column slot"""
    col = np.asarray(col, np.int64)
    return ((col // maxpart) * grid_cols + grid_c) * maxpart + col % maxpart


def push_reference(rows, cols, n_rows, frontier, visited, maxpart, grid_cols, grid_c):
    """cugraph_b200_block_bfs_push restated: the largest code of a frontier source of every unvisited row, else -1"""
    want = np.full(n_rows, -1, np.int64)
    live = (frontier[cols] != 0) & (visited[rows] == 0)
    np.maximum.at(want, rows[live], code_of(cols[live], maxpart, grid_cols, grid_c))
    return want


def bottom_up_reference(alpha, beta, now, n_f, prev_n_f, m_f, m_u, n_unvisited):
    """Beamer's rule as run_bfs (traverse.cu) applies it"""
    if not now and m_f * alpha > m_u and n_f >= prev_n_f:
        return True
    if now and n_f * beta < n_unvisited and n_f < prev_n_f:
        return False
    return now


class Block:
    """one cugraph_b200 block of (rows, cols) on a fresh handle, freed by close()"""

    def __init__(self, rows, cols, n_rows, n_cols, device="cpu"):
        import torch
        from cugraph_b200 import _capi
        from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
        from cugraph_b200.pylibcugraph.utils import View
        self.L, self.capi = _capi.lib(), _capi
        self.handle = ResourceHandle(stream=torch.cuda.current_stream().cuda_stream if device != "cpu" else 0)
        r, c = View(torch.as_tensor(rows).to(device)), View(torch.as_tensor(cols).to(device))
        blk, err = C.c_void_p(), C.c_void_p()
        try:
            code = self.L.cugraph_b200_block_create(self.handle.ptr, n_rows, n_cols, r.ptr, c.ptr, None, C.byref(blk), C.byref(err))
            _capi.check(code, err, "cugraph_b200_block_create")
        finally:
            r.free()
            c.free()
        self.ptr = blk.value

    def call(self, name, *args):
        """self.L.<name>(handle, block, *args, &error): tensors are passed as views"""
        import torch
        from cugraph_b200.pylibcugraph.utils import View
        views, a = [], []
        for x in args:
            if isinstance(x, torch.Tensor):
                views.append(View(x))
                a.append(views[-1].ptr)
            else:
                a.append(x)
        err = C.c_void_p()
        try:
            code = getattr(self.L, name)(self.handle.ptr, self.ptr, *a, C.byref(err))
            self.capi.check(code, err, name)
        finally:
            for v in views:
                v.free()

    def close(self):
        self.L.cugraph_b200_block_free(self.ptr)
