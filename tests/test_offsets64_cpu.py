"""64-bit row offsets on the CPU.  By default only a graph of 2^31 or more edges gets them; CUGRAPH_B200_OFFS64_MIN_EDGES=0
gives them to every graph, so that the int64_t instantiations of staging and of every algorithm run on small graphs.

Staging: the emulated library's primary orientation with 64-bit offsets holds the same offsets, indices, weights, segment
bounds and nnz_hi as the default build of the same graph.  Algorithms: the checks of tests/test_paths_gpu.py, driven through
the Python surface over the emulation build of the library (tests/emu_py.py), against the oracle and against the default
run of the same graph."""
import ctypes as C

import numpy as np
import pytest

from tests import test_paths_gpu as paths
from tests.emu_py import surface  # noqa: F401
from tests.test_emu_staging_cpu import create_graph, emu, make_edges, primary  # noqa: F401


@pytest.mark.parametrize("weighted", [False, True])
def test_staging_offs64_matches_default(emu, monkeypatch, weighted):  # noqa: F811
    src, dst, w = make_edges(20_000, 150_000, seed=31 + weighted, weighted=weighted, id_offset=11)
    g = create_graph(emu, src, dst, w)
    P32 = primary(emu, g)
    assert not P32["offs64"] and P32["off"].dtype == np.int32
    for knob in ("0", "-5", "150000"):             # below zero clamps to 0; at the edge count the offsets widen
        monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", knob)
        g64 = create_graph(emu, src, dst, w)
        P64 = primary(emu, g64)
        assert P64["offs64"] and P64["off"].dtype == np.int64, knob
        assert np.array_equal(P64["off"], P32["off"]) and np.array_equal(P64["idx"], P32["idx"])
        assert (P64["w"] is None) == (w is None) and (w is None or np.array_equal(P64["w"], P32["w"]))
        assert P64["seg"] == P32["seg"] and P64["nnz_hi"] == P32["nnz_hi"] and np.array_equal(P64["ext"], P32["ext"])
        emu.cugraph_graph_free(g64)
    for knob in ("150001", str(1 << 40)):          # above the edge count, and clamped to 2^31: 32-bit offsets
        monkeypatch.setenv("CUGRAPH_B200_OFFS64_MIN_EDGES", knob)
        g32 = create_graph(emu, src, dst, w)
        assert not primary(emu, g32)["offs64"], knob
        emu.cugraph_graph_free(g32)
    monkeypatch.delenv("CUGRAPH_B200_OFFS64_MIN_EDGES")
    emu.emu_reload_tuning(C.c_void_p(emu.handle))
    emu.cugraph_graph_free(g)


SCALE = 9


@pytest.mark.parametrize("directions", [(False,), (True,)], ids=["top-down", "direction-optimizing"])
def test_bfs_offs64_emulated(surface, monkeypatch, directions):
    paths.check_bfs(monkeypatch, paths.OFFS64, SCALE, directions=directions)


def test_sssp_offs64_emulated(surface, monkeypatch):
    paths.check_sssp(monkeypatch, paths.OFFS64, SCALE)


@pytest.mark.parametrize("wdtype", [np.float32, np.float64])
def test_sssp_offs64_zero_weight_predecessors_emulated(surface, monkeypatch, wdtype):
    paths.check_sssp_zero_weights(monkeypatch, paths.OFFS64, wdtype)


def test_advance_in_halves_offs64_emulated(surface, monkeypatch):
    knobs = {**paths.OFFS64, "ADVANCE_SPLIT_EDGES": "500"}
    paths.check_bfs(monkeypatch, knobs, SCALE, depth_limit=False)
    paths.check_sssp(monkeypatch, knobs, SCALE, cutoff=False, no_pred=False)


@pytest.mark.parametrize("store_transposed", [True, False])
def test_pagerank_offs64_emulated(surface, monkeypatch, store_transposed):
    paths.check_pagerank_offs64(monkeypatch, SCALE, store_transposed, weighted=store_transposed)


def test_katz_hits_eigenvector_offs64_emulated(surface, monkeypatch):
    paths.check_siblings(monkeypatch, paths.OFFS64, SCALE)


def test_wcc_degrees_extract_paths_offs64_emulated(surface, monkeypatch):
    paths.check_structure(monkeypatch, paths.OFFS64, SCALE)


def test_csr_input_offs64_emulated(surface, monkeypatch):
    paths.check_csr_input(monkeypatch, paths.OFFS64)


def test_int64_ids_double_weights_offs64_emulated(surface, monkeypatch):
    paths.check_int64_ids_double_weights(monkeypatch, paths.OFFS64)
