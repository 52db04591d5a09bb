"""The driver checks of tests/sweep_drivers.py on the CPU, over the emulation build of the library (tests/emu_py.py): Katz,
eigenvector centrality, HITS and personalized PageRank step for step against their fp64 references on every sweep layout
and element type at RMAT-9, the other orientations, one graph through many calls and PageRank's expensive input checks.
The emulation runs CTAs one after another, so this checks the drivers' logic and the layouts, not their concurrency."""
import pytest

from tests import sweep_drivers as sd
from tests import test_sweep_drivers_gpu as gpu
from tests.emu_py import surface  # noqa: F401

SCALE = {"f32w": 9, "f64w": 9, "f32": 9}


@pytest.mark.parametrize("etype", list(SCALE))
@pytest.mark.parametrize("layout", list(sd.KNOBS))
@pytest.mark.parametrize("algorithm", gpu.ALGORITHMS)
def test_driver_layouts_emulated(surface, monkeypatch, capfd, algorithm, layout, etype):  # noqa: F811
    sd.run_case(algorithm, monkeypatch, capfd, sd.graph_of(etype, SCALE[etype]), layout)


@pytest.mark.parametrize("orientation", ["csr", "symmetric", "csr-input"])
@pytest.mark.parametrize("algorithm", gpu.ALGORITHMS)
def test_driver_orientations_emulated(surface, monkeypatch, capfd, algorithm, orientation):  # noqa: F811
    sd.run_case(algorithm, monkeypatch, capfd, sd.graph_of("f32w", 9, orientation), "bands-tail")


def test_driver_scattered_int64_ids_emulated(surface, monkeypatch, capfd):  # noqa: F811
    for algorithm in gpu.ALGORITHMS:
        sd.run_case(algorithm, monkeypatch, capfd, sd.graph_of("f64w", 9, "csr", scattered_ids=True), "bands-tail")


@pytest.mark.parametrize("orientation", ["csc", "csr"])
def test_one_graph_many_calls_emulated(surface, monkeypatch, capfd, orientation):  # noqa: F811
    sd.run_many_calls(monkeypatch, capfd, sd.graph_of("f32w", 9, orientation), "bands-tail")


def test_edge_cases_emulated(surface, monkeypatch, capfd):  # noqa: F811
    gpu.test_isolated_vertices_only(monkeypatch, capfd)
    gpu.test_single_self_loop(monkeypatch, capfd)
    gpu.test_too_few_iterations(monkeypatch, capfd)


@pytest.mark.parametrize("T", [sd.np.float32, sd.np.float64])
def test_pagerank_expensive_checks_emulated(surface, monkeypatch, T):  # noqa: F811
    gpu.test_pagerank_expensive_checks(monkeypatch, T)
    gpu.test_pagerank_expensive_checks_pass_valid_inputs(monkeypatch, T)
