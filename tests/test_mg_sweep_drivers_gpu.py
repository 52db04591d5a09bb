"""Multi-GPU PageRank, Katz, eigenvector centrality and HITS on the H100, step for step against fp64 references
(tests/mg_sweep_drivers.py, the bounds of tests/sweep_drivers.py with the reduce-scatter's rounding added), on every grid
and every block sweep layout: the plain sweep, the piece stream, the piece stream in bands with a tail, and 64-bit offsets.
float32 weights and unweighted on directed RMAT-18, float64 weights on RMAT-17 (a block's columns span more than one
192 KiB shared-memory slice on the 2x2 grid), multi-edges and self-loops kept; scattered int64 ids; one graph through
many calls; NCCL process groups of 1, 2 and 4 GPUs; and, without knobs, RMAT-21 on 2x2, where every block is past the
piece stream's edge threshold.  The worst observed / bound per algorithm, type and grid is printed at the end."""
import numpy as np
import pytest

from tests import mg_sweep_drivers as msd
from tests import sweep_drivers as sd
from tests import sweep_rows as sr

pytestmark = pytest.mark.gpu

SCALE = {"f32w": 18, "f64w": 17, "f32": 18}


@pytest.fixture(scope="module", autouse=True)
def report_margins(request):
    yield
    msd.report(request, "worst |got - ref| / bound per algorithm, element type and grid (multi-GPU):")


@pytest.mark.parametrize("etype", list(SCALE))
@pytest.mark.parametrize("layout", list(sd.KNOBS))
@pytest.mark.parametrize("grid", list(msd.GRIDS))
def test_mg_driver_layouts(monkeypatch, capfd, grid, layout, etype):
    graph = msd.graph_of(etype, SCALE[etype])
    _, blocks = msd.run(monkeypatch, capfd, graph, layout, grid, msd.all_calls(graph, 30))
    if grid == "2x2" and layout in ("stream", "bands-tail"):
        # x spans more than one shared-memory slice: the piece stream runs over several column blocks
        assert all(w["B"] >= 2 for _, ws in blocks for w in ws), blocks


def test_mg_driver_scattered_int64_ids(monkeypatch, capfd):
    graph = msd.graph_of("f64w", SCALE["f64w"], scattered_ids=True)
    msd.run(monkeypatch, capfd, graph, "bands-tail", "2x2", msd.all_calls(graph, 30))


@pytest.mark.parametrize("layout", ["bands-tail", "plain"])
def test_mg_one_graph_many_calls(monkeypatch, capfd, layout):
    """state a block carries from one driver to the next: the y arrays' written rows, the transposed copy HITS builds"""
    graph = msd.graph_of("f32w", SCALE["f32w"])
    msd.run(monkeypatch, capfd, graph, layout, "2x2", msd.many_calls(graph))


@pytest.mark.parametrize("world", [1, 2, 4])
@pytest.mark.parametrize("layout", ["bands-tail", "plain"])
def test_mg_drivers_nccl(monkeypatch, capfd, layout, world):
    """the real collectives and stream ordering: PageRank's totals all-reduced while the next sweep runs; 2 and 4 GPUs are
    skipped when fewer are visible"""
    graph = msd.graph_of("f32w", SCALE["f32w"])
    msd.run(monkeypatch, capfd, graph, layout, f"nccl-{world}", msd.all_calls(graph, 30))


def test_mg_drivers_production_layout(monkeypatch, capfd):
    """no knobs: RMAT-21 (device generator) on 2x2 puts every block past the piece stream's 2^22 edges, so each runs the
    default piece stream, in bands sized by the L2"""
    from cugraph_b200 import generators
    scale = 21
    s, d = generators.rmat_edgelist(scale, 16 << scale, seed=2100)
    s, d = s.cpu().numpy().astype(np.int64), d.cpu().numpy().astype(np.int64)
    graph = msd.over_present(s, d, np.float32, None, label=f"RMAT-{scale} float32 (device generator)")
    del s, d
    calls = [dict(algo="pagerank", steps=30), msd.katz_calls(graph)[0]]
    _, blocks = msd.run(monkeypatch, capfd, graph, "default", "2x2", calls)
    # the traces matched sweep_rows.expected_layout without knobs: the bands are those the L2 size gives
    assert all(nnz >= sr.DEFAULT_MIN_EDGES and ws[0] is not None for nnz, ws in blocks), blocks
