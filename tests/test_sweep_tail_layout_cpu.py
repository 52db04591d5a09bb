"""The tail layout (sweep_layout.cuh, sweep_layout.cu): the rows of in-degree below the bound, in runs of equal in-degree cut into
tiles of 32 rows whose ids are lane-interleaved.  Checked on the CPU with forced bounds: the runs tile [n_str, n_cov) with one
in-degree each, every (row, source[, weight]) of the tail sits exactly where the layout says, in the row's order, padding
(column n_vertices, weight 0) only in the last tile of a run; and PageRank and the emulated 2D multi-GPU block sweep through
the tail kernel match their references."""
import ctypes as C

import numpy as np
import pytest

import oracle
from tests.emu_py import surface  # noqa: F401
from tests.test_emu_algorithms_cpu import dense_ids, run_pagerank
from tests.test_emu_mg_cpu import test_2d_partitioned_pagerank_on_one_cpu as mg_case
from tests.test_emu_staging_cpu import as_np, create_graph, emu, make_edges, primary  # noqa: F401
from tests.test_sweep_bands_cpu import layout_arrays
from tests.test_sweep_tail_cpu import THRESHOLDS, stream_rows

TILE = 32
UNIT_ENTRIES = 24   # kTailUnitEntries


def unit_tiles(d):
    return max(1, UNIT_ENTRIES // d)


def tail_of(L, g, es):
    L.emu_sweep_tail.restype = C.c_int
    L.emu_sweep_tail.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    cap = 64
    runs = np.zeros((cap, 5), dtype=np.int64)
    ptrs = (C.c_void_p * 2)()
    n = L.emu_sweep_tail(g, es, runs.ctypes.data, cap, ptrs)
    assert 0 < n < cap
    return runs[:n + 1], ptrs


@pytest.mark.parametrize("bound", [2, 8, 16, 32])
@pytest.mark.parametrize("weighted", [False, True])
def test_tail_runs_and_tiles(emu, monkeypatch, bound, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", str(bound))
    src, dst, w = make_edges(120_000, 900_000, seed=71 + bound + weighted, weighted=weighted, id_offset=3)
    g = create_graph(emu, src, dst, w)
    P = primary(emu, g)
    A = layout_arrays(emu, g)
    n_cov, n_str = P["seg"][5], stream_rows(emu, g, A["es"])
    assert n_str == P["seg"][THRESHOLDS.index(bound)] and 0 < n_str < n_cov
    runs, ptrs = tail_of(emu, g, A["es"])
    deg = np.diff(P["off"]).astype(np.int64)
    # the runs tile [n_str, n_cov), one in-degree each, descending
    assert runs[0, 1] == n_str and runs[-1, 1] == n_cov and runs[-1, 0] == 0
    assert (np.diff(runs[:-1, 0]) < 0).all() and (runs[:-1, 0] >= 1).all() and (runs[:-1, 0] < bound).all()
    assert runs[0, 2] == 0 and runs[0, 3] == 0 and runs[0, 4] == 0
    n_ids = int(runs[-1, 4])
    ids = as_np(ptrs[0], n_ids, np.int32)
    tw = as_np(ptrs[1], n_ids, np.float32) if weighted else None
    seen = 0
    for (d, r0, t0, u0, o0), (_, r1, t1, u1, o1) in zip(runs[:-1], runs[1:]):
        assert r1 > r0 and (deg[r0:r1] == d).all()
        tiles = -(-(r1 - r0) // TILE)
        assert t1 - t0 == tiles and u1 - u0 == -(-tiles // unit_tiles(d)) and o1 - o0 == tiles * TILE * d
        # entry k of lane l of tile t at o0 + t * 32 * d + k * 32 + l
        got = ids[o0:o1].reshape(tiles, d, TILE).transpose(0, 2, 1).reshape(tiles * TILE, d)
        rows = np.arange(r0, r0 + tiles * TILE)
        live = rows < r1
        assert (~live).sum() < TILE and live[:(tiles - 1) * TILE].all()  # padding: the run's last tile only
        e = P["off"][rows[live]][:, None].astype(np.int64) + np.arange(d)[None, :]
        assert np.array_equal(got[live], P["idx"][e])                   # every entry of a row, in the row's order
        assert (got[~live] == P["nv"]).all()                             # padding reads x[n_vertices] = 0
        if weighted:
            gw = tw[o0:o1].reshape(tiles, d, TILE).transpose(0, 2, 1).reshape(tiles * TILE, d)
            assert np.array_equal(gw[live], P["w"][e]) and (gw[~live] == 0).all()
        seen += int(live.sum()) * d
    assert seen == int(P["off"][n_cov] - P["off"][n_str])               # each tail edge exactly once
    emu.cugraph_graph_free(g)


@pytest.mark.parametrize("bound,weighted", [(2, False), (16, False), (16, True), (32, True)])
def test_pagerank_through_tail_kernel(emu, monkeypatch, bound, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", str(bound))
    src, dst, w = make_edges(60_000, 250_000, seed=150 + bound + weighted, weighted=weighted, id_offset=2)
    g = create_graph(emu, src, dst, w)
    verts, pr, it = run_pagerank(emu, g, 0.85, 0.0, 20)
    P = primary(emu, g)
    A = layout_arrays(emu, g)
    assert 0 < stream_rows(emu, g, A["es"]) < P["seg"][5]
    ids, s, d = dense_ids(src, dst)
    ref, _, _ = oracle.pagerank(s, d, ids.size, None if w is None else w.astype(np.float64), alpha=0.85, epsilon=0.0,
                                max_iterations=20)
    assert it == 20
    got = np.zeros(ids.size)
    got[np.searchsorted(ids, verts)] = pr
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)
    emu.cugraph_graph_free(g)


@pytest.mark.parametrize("R,Cc,weighted", [(2, 2, True), (2, 4, False)])
def test_mg_blocks_with_tail_bound_16(surface, monkeypatch, R, Cc, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", "16")
    mg_case(surface, monkeypatch, R, Cc, weighted, "0")
