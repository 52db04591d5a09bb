"""The tail of the piece stream (sweep_layout.cu, sweep.cuh): rows of in-degree below a bound leave the stream and are swept
by the plain row kernel after the bands.  Checked on the CPU with forced bounds (CUGRAPH_B200_SWEEP_TAIL_DEGREE): the stream
holds exactly the edges of the rows [0, n_str), each once, and its bands partition [0, n_str); bound 1 is the layout without
a tail; PageRank, Katz, HITS, the plain-vs-stream row comparison and the emulated 2D multi-GPU block sweep all match their
references with a tail."""
import ctypes as C

import numpy as np
import pytest

import oracle
from tests.emu_py import surface  # noqa: F401
from tests.test_emu_algorithms_cpu import dense_ids, run_pagerank
from tests.test_emu_algorithms_cpu import test_sweep_against_plain_sweep_emulated as compare_sweeps_case
from tests.test_emu_mg_cpu import test_2d_partitioned_pagerank_on_one_cpu as mg_case
from tests.test_emu_siblings_cpu import test_hits_emulated as hits_case
from tests.test_emu_siblings_cpu import test_katz_emulated as katz_case
from tests.test_emu_staging_cpu import create_graph, emu, make_edges, primary, sweep_pieces  # noqa: F401
from tests.test_sweep_bands_cpu import bands_of, layout_arrays

THRESHOLDS = (32, 16, 8, 4, 2, 1, 0)   # kSegThreshold: seg[k] = rows of in-degree >= THRESHOLDS[k]


def stream_rows(L, g, es):
    L.emu_sweep_stream_rows.restype = C.c_int32
    L.emu_sweep_stream_rows.argtypes = [C.c_void_p, C.c_size_t]
    return int(L.emu_sweep_stream_rows(g, es))


@pytest.mark.parametrize("bound,weighted,bands", [(2, False, "0"), (2, True, "3"), (8, False, "3"), (8, True, "0"),
                                                  (32, False, "0"), (32, True, "2")])
def test_tail_layout(emu, monkeypatch, bound, weighted, bands):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", str(bound))
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_BANDS", bands)
    src, dst, w = make_edges(120_000, 900_000, seed=13 + bound + weighted, weighted=weighted, id_offset=7)
    g = create_graph(emu, src, dst, w)
    P = primary(emu, g)
    H = sweep_pieces(emu, g, P)                          # structural checks of every chunk, and the decoded entries
    A = layout_arrays(emu, g)
    n_cov, n_str = P["seg"][5], stream_rows(emu, g, A["es"])
    assert n_str == P["seg"][THRESHOLDS.index(bound)] and 0 < n_str < n_cov
    # exactly the edges of the rows [0, n_str), each once
    e_str = int(P["off"][n_str])
    rows = np.repeat(np.arange(n_str), np.diff(P["off"][:n_str + 1]))
    cols = P["idx"][:e_str].astype(np.int64)
    assert H["r"].size == e_str and (H["r"] < n_str).all()
    if P["w"] is None:
        o1, o2 = np.lexsort((H["c"], H["r"])), np.lexsort((cols, rows))
        assert (H["r"][o1] == rows[o2]).all() and (H["c"][o1] == cols[o2]).all()
    else:
        o1, o2 = np.lexsort((H["w"], H["c"], H["r"])), np.lexsort((P["w"][:e_str], cols, rows))
        assert (H["r"][o1] == rows[o2]).all() and (H["c"][o1] == cols[o2]).all() and (H["w"][o1] == P["w"][:e_str][o2]).all()
    # the bands partition [0, n_str)
    n_bands, _, band_row, _ = bands_of(emu, g, A["es"], A["n_cta_flat"])
    assert band_row[0] == 0 and band_row[-1] == n_str and (np.diff(band_row) > 0).all() and (band_row[:-1] % 512 == 0).all()
    if bands != "0":
        assert n_bands == min(int(bands), -(-n_str // 512))
    emu.cugraph_graph_free(g)


@pytest.mark.parametrize("weighted", [False, True])
def test_bound_one_is_the_layout_without_tail(emu, monkeypatch, weighted):  # noqa: F811
    """on graphs below the default's edge count the default has no tail either: bound 1 must give the same layout, array for
    array"""
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    src, dst, w = make_edges(120_000, 900_000, seed=31 + weighted, weighted=weighted, id_offset=1)
    got = {}
    for bound in (None, "1"):
        if bound is None:
            monkeypatch.delenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", raising=False)
        else:
            monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", bound)
        g = create_graph(emu, src, dst, w)
        P = primary(emu, g)
        A = layout_arrays(emu, g)
        assert stream_rows(emu, g, A["es"]) == P["seg"][5]
        got[bound] = A
        emu.cugraph_graph_free(g)
    for k in ("rows", "chunks", "phases", "cta"):
        assert np.array_equal(got[None][k], got["1"][k]), k


@pytest.mark.parametrize("bound", [4, 8, 32])
@pytest.mark.parametrize("bands", [1, 3])
def test_pagerank_with_tail_emulated(emu, monkeypatch, bound, bands):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", str(bound))
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_BANDS", str(bands))
    weighted = bound == 8
    src, dst, w = make_edges(60_000, 250_000, seed=90 + bound, weighted=weighted, id_offset=4)
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


@pytest.mark.parametrize("weighted", [False, True])
def test_stream_with_tail_against_plain_sweep(emu, monkeypatch, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", "8")
    compare_sweeps_case(emu, monkeypatch, weighted)


@pytest.mark.parametrize("weighted", [False, True])
def test_katz_with_tail(emu, monkeypatch, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", "8")
    katz_case(emu, monkeypatch, weighted, "0")


@pytest.mark.parametrize("transposed,weighted,normalize,guess", [(False, False, True, False), (True, True, False, True)])
def test_hits_with_tail(emu, monkeypatch, transposed, weighted, normalize, guess):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", "8")
    emu.emu_reload_tuning(C.c_void_p(emu.handle))
    hits_case(emu, transposed, weighted, normalize, guess)
    monkeypatch.undo()
    emu.emu_reload_tuning(C.c_void_p(emu.handle))


@pytest.mark.parametrize("R,Cc,weighted", [(2, 2, False), (2, 4, True)])
def test_mg_blocks_with_tail(surface, monkeypatch, R, Cc, weighted):  # noqa: F811
    """covered_rows_only + row_vertex: the block sweep leaves the empty rows of y alone, the tail writes its rows"""
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", "4")
    mg_case(surface, monkeypatch, R, Cc, weighted, "0")
