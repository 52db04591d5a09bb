"""Multi-GPU multi-source BFS (MGGraph.multi_source_bfs) on every rank of a grid in ONE process (tests/mg_world.py), the
checks of its rows, and numpy restatements of its five entry points: cugraph_b200_block_ms_bfs_push / _pull / _pred on one
block and cugraph_b200_ms_bfs_owner_step / _owner_pred.  The graphs and schedules are tests/mg_bfs_direction_ref.py's.

Shared by tests/test_mg_multi_source_bfs_cpu.py and tests/test_mg_multi_source_bfs_gpu.py."""
import numpy as np

import oracle
from tests import mg_bfs_direction_ref as dref
from tests import mg_paths_ref as refs
from tests import mg_world

IMAX = refs.IMAX
SOURCE_COUNTS = (1, 63, 64, 65, 130)


def pick_sources(case, n, rng):
    """n source indices of the case (vertices of its edges), the last one repeating the first (a duplicate row)"""
    ids = np.unique(np.concatenate([case.s, case.d]))
    src = rng.choice(ids, n).astype(np.int64)
    if n > 1:
        src[-1] = src[0]
    return src


def checked_rows(n):
    """the rows compared with a BFS of their own: the first, the first of the second batch and the last"""
    return sorted({0, min(64, n - 1), n - 1}) if n else []


def _ext(case, a):
    """indices -> the case's external ids"""
    return a if case.ids is None else case.ids[np.asarray(a, np.int64)]


def _worker(rank, world, case, sources, do, limit, dests, device):
    import torch
    g = mg_world.graph(rank, world, _ext(case, case.s), _ext(case, case.d), device=device)
    order = None if case.ids is None else np.argsort(case.ids)

    def index(x):   # external ids -> indices (-1 stays -1)
        x = x.cpu().numpy().astype(np.int64)
        if order is None:
            return x
        pos = np.searchsorted(case.ids[order], np.where(x >= 0, x, case.ids.min())).clip(max=order.size - 1)
        return np.where(x >= 0, order[pos], -1)

    vdt = torch.int64 if case.ids is not None else torch.int32
    src = torch.as_tensor(_ext(case, sources)).to(vdt).to(device)
    v, dist, pred = g.multi_source_bfs(src, limit, direction_optimizing=do)
    out = dict(v=index(v), dist=dist.cpu().numpy(), pred=index(pred.reshape(-1)).reshape(pred.shape),
               n_local=g.part.n_local, stats=dict(g.last_ms_bfs_stats), rows={})
    for k in checked_rows(len(sources)):
        s_k = int(src[k])
        _, d1, p1 = g.bfs(s_k, limit)                       # the default top-down schedule
        row = dict(dist=bool(torch.equal(dist[k], d1)), pred=bool(torch.equal(pred[k], p1)),
                   valid=g.validate_bfs(v, dist[k], pred[k], s_k, limit)["ok"])
        if limit < 0:
            dst = torch.as_tensor(_ext(case, dests[rank])).to(vdt).to(device)
            pa, la = g.extract_paths(dist[k], pred[k], dst)
            pb, lb = g.extract_paths(d1, p1, dst)
            row["paths"] = la == lb and bool(torch.equal(pa, pb))
        out["rows"][k] = row
    return out


def gather(res):
    """(vertex indices, distances [n, V], predecessor indices [n, V], codes [V]) over the ranks; a vertex's code is owner
    rank * maxpart + local id, maxpart the largest n_local"""
    mp = max(max(r["n_local"] for r in res), 1)
    vids = np.concatenate([r["v"] for r in res]).astype(np.int64)
    dist = np.concatenate([r["dist"] for r in res], axis=1)
    pred = np.concatenate([r["pred"] for r in res], axis=1).astype(np.int64)
    codes = np.concatenate([rank * mp + np.arange(r["n_local"]) for rank, r in enumerate(res)]).astype(np.int64)
    return vids, dist, pred, codes


def check_rows(s, d, res, sources, depth_limit=-1, vertices=()):
    """every row k against the oracle BFS from sources[k] on the vertices of the edges and `vertices`: distances bit-exact,
    and predecessors by the rule of the top-down MGGraph.bfs: the in-neighbour one level closer with the largest code.
    Returns the rows' largest finite distances."""
    vids, dist, pred, codes = gather(res)
    ids = np.unique(np.concatenate([np.asarray(x, np.int64) for x in (s, d, vertices)]))
    remap = np.full(int(ids.max(initial=0)) + 1, -1, np.int64)
    remap[ids] = np.arange(ids.size)
    assert np.array_equal(np.sort(vids), ids)
    assert dist.shape == pred.shape == (len(sources), ids.size)
    col = remap[vids]
    code_by = np.empty(ids.size, np.int64)
    code_by[col] = codes
    rs, rd = remap[s], remap[d]
    csr = oracle.coo_to_csx(rs.astype(np.int32), rd.astype(np.int32), ids.size)
    ecc = []
    for k, src in enumerate(np.asarray(sources, np.int64)):
        ref_d, _ = oracle.bfs(rs, rd, ids.size, [int(remap[src])], depth_limit=None if depth_limit < 0 else depth_limit, csr=csr)
        ref_d = np.asarray(ref_d, np.int64)
        ref_d = np.where((ref_d < 0) | (ref_d >= IMAX), IMAX, ref_d)
        if depth_limit == 0:   # MGGraph.bfs runs no level (the oracle always runs one)
            ref_d = np.where(ref_d == 0, 0, IMAX)
        got_d = np.empty(ids.size, np.int64)
        got_d[col] = dist[k]
        assert np.array_equal(got_d, ref_d), k
        want = np.full(ids.size, -1, np.int64)
        e = (ref_d[rs] < IMAX) & (ref_d[rs] + 1 == ref_d[rd])
        np.maximum.at(want, rd[e], code_by[rs[e]])
        got_p = np.full(ids.size, -1, np.int64)
        got_p[col] = np.where(pred[k] >= 0, code_by[remap[np.maximum(pred[k], 0)]], -1)
        assert np.array_equal(got_p, want), k
        ecc.append(int(ref_d[ref_d < IMAX].max()))
    return ecc


def expected_levels(ecc, depth_limit):
    """the levels a run takes: per batch of 64, its largest distance + 1 (the last level finds nothing), capped by the limit"""
    total = 0
    for b0 in range(0, len(ecc), 64):
        top = max(ecc[b0:b0 + 64]) + 1
        total += top if depth_limit < 0 else min(top, depth_limit)
    return total


def run_case(case, world, schedule, n_sources, depth_limit, rng, device="cpu"):
    """MGGraph.multi_source_bfs on `world` ranks (the grid and knobs set by the caller) from n_sources of the case's
    vertices; every check of the module"""
    do, _ = dref.SCHEDULES[schedule]
    sources = pick_sources(case, n_sources, rng)
    ids = np.unique(np.concatenate([case.s, case.d]))
    dests = refs.split(rng.choice(ids, 12), world, rng)
    res = mg_world.run(world, _worker, case, sources, do, depth_limit, dests, device)
    what = f"{case.name} {schedule} n={n_sources} depth_limit={depth_limit}"
    ecc = check_rows(case.s, case.d, res, sources, depth_limit)
    st = res[0]["stats"]
    assert all(r["stats"] == st for r in res), what
    assert st["batches"] == -(-n_sources // 64), what
    assert st["levels"] == expected_levels(ecc, depth_limit) == st["top_down"] + st["bottom_up"], (what, st)
    if not do:
        assert st["bottom_up"] == 0, what
    for r in res:
        for k, row in r["rows"].items():
            assert all(row.values()), (what, k, row)


# ---------------------------------------------------------------------------------------------------- entry points
def _bits(words):
    return np.asarray(words, np.int64).view(np.uint64)


def step_reference(rows, cols, n_rows, cur, seen, n_sources):
    """cugraph_b200_block_ms_bfs_push / _pull restated: next[row] = OR over the row's columns of cur & ~seen & mask"""
    mask = np.uint64(0xFFFFFFFFFFFFFFFF if n_sources == 64 else (1 << n_sources) - 1)
    cur, seen = _bits(cur), _bits(seen)
    out = np.zeros(n_rows, np.uint64)
    np.bitwise_or.at(out, rows, cur[cols] & ~seen[rows] & mask)
    return out.view(np.int64)


def pred_reference(rows, cols, n_rows, cur, new_rows, maxpart, grid_cols, grid_c, seg):
    """cugraph_b200_block_ms_bfs_pred restated: the largest code of a column with the bit, per (row, bit), in the padded
    owner segments"""
    cur, new = _bits(cur), _bits(new_rows)
    pairs = np.full(grid_cols * seg, -1, np.int64)
    pc = np.array([bin(int(x)).count("1") for x in new], np.int64)
    code = dref.code_of(cols, maxpart, grid_cols, grid_c)
    for r in np.flatnonzero(new):
        k = r // maxpart
        base = k * seg + pc[k * maxpart:r].sum()
        b = int(new[r])
        e = rows == r
        for j in range(64):
            if not (b >> j) & 1:
                continue
            has = e & (((cur[cols] >> np.uint64(j)) & np.uint64(1)) != 0)
            pos = base + bin(b & ((1 << j) - 1)).count("1")
            if has.any() and pos < (k + 1) * seg:
                pairs[pos] = code[has].max()
    return pairs


def owner_step_reference(recv, parts, maxpart, n_local, n_sources, level, seen, cur, dist, deg_out, deg_in):
    """cugraph_b200_ms_bfs_owner_step restated: (seen, cur, dist, counts) after the step"""
    mask = np.uint64(0xFFFFFFFFFFFFFFFF if n_sources == 64 else (1 << n_sources) - 1)
    r = _bits(recv)[:parts * maxpart].reshape(parts, maxpart)[:, :n_local]
    nxt = np.bitwise_or.reduce(r, axis=0) if parts else np.zeros(n_local, np.uint64)
    seen, cur, dist = _bits(seen).copy(), _bits(cur).copy(), np.array(dist, np.int32).reshape(n_sources, -1).copy()
    s = seen[:n_local]
    nw = nxt & ~s & mask
    cur[:n_local] = nw
    seen[:n_local] = s | nw
    for j in range(n_sources):
        dist[j, ((nw >> np.uint64(j)) & np.uint64(1)) != 0] = level
    has = nw != 0
    full = has & ((s | nw) == mask)
    dout = np.zeros(n_local, np.int64) if deg_out is None else np.asarray(deg_out)[:n_local]
    din = np.zeros(n_local, np.int64) if deg_in is None else np.asarray(deg_in)[:n_local]
    counts = [has.sum(), dout[has].sum(), full.sum(), din[full].sum(), sum(bin(int(x)).count("1") for x in nw)]
    return seen.view(np.int64), cur.view(np.int64), dist.reshape(-1), np.asarray(counts, np.int64)


def owner_pred_reference(new_words, pairs, n_local, n_sources, pred):
    """cugraph_b200_ms_bfs_owner_pred restated"""
    nw = _bits(new_words)[:n_local]
    out = np.array(pred, np.int64).reshape(n_sources, -1).copy()
    at = 0
    for v in range(n_local):
        b = int(nw[v])
        for j in range(64):
            if (b >> j) & 1:
                if at < len(pairs):
                    out[j, v] = pairs[at]
                at += 1
    return out.reshape(-1)
