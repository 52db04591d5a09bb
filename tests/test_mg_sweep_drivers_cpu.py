"""The multi-GPU driver checks of tests/mg_sweep_drivers.py on the CPU, over the emulation build of the library
(tests/emu_py.py): MGGraph's PageRank, Katz, eigenvector centrality and HITS step for step against their fp64 references
at RMAT-10 under the plain sweep, the piece stream and the piece stream in bands with a tail, on the simulated grids 1x2,
2x2 and 4x2 and a gloo process group of 2; scattered int64 ids and one graph through many calls.  The emulation runs CTAs one after another, so this
checks the drivers' logic, the exchange and the layouts, not their concurrency."""
import pytest

from tests import mg_sweep_drivers as msd
from tests.emu_py import surface  # noqa: F401

SCALE = 10
STEPS = 10                   # the emulation runs a launch's threads one after the other


@pytest.fixture(scope="module", autouse=True)
def report_margins(request):
    yield
    msd.report(request, "worst |got - ref| / bound per algorithm, element type and grid (multi-GPU, emulated):")


@pytest.mark.parametrize("etype", ["f32w", "f64w", "f32"])
@pytest.mark.parametrize("layout", ["plain", "stream", "bands-tail"])
def test_mg_driver_layouts_emulated(surface, monkeypatch, capfd, layout, etype):  # noqa: F811
    graph = msd.graph_of(etype, SCALE)
    msd.run(monkeypatch, capfd, graph, layout, "2x2", msd.all_calls(graph, STEPS))


@pytest.mark.parametrize("grid", ["1x2", "4x2", "gloo-2"])
def test_mg_driver_grids_emulated(surface, monkeypatch, capfd, grid):  # noqa: F811
    graph = msd.graph_of("f32w", SCALE)
    msd.run(monkeypatch, capfd, graph, "bands-tail", grid, msd.all_calls(graph, STEPS))


def test_mg_driver_scattered_int64_ids_emulated(surface, monkeypatch, capfd):  # noqa: F811
    graph = msd.graph_of("f64w", SCALE, scattered_ids=True)
    msd.run(monkeypatch, capfd, graph, "bands-tail", "2x2", msd.all_calls(graph, STEPS))


def test_mg_one_graph_many_calls_emulated(surface, monkeypatch, capfd):  # noqa: F811
    graph = msd.graph_of("f32w", SCALE)
    msd.run(monkeypatch, capfd, graph, "bands-tail", "2x2", msd.many_calls(graph, STEPS))
