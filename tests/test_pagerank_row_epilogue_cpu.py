"""The checks of tests/test_pagerank_row_epilogue_gpu.py on the CPU, over the emulation build of the library
(tests/emu_py.py): PageRank with the sweep's row epilogue against its fp64 restatement on every sweep layout and element
type at RMAT-9, its launches per iteration, and a small graph of dangling and isolated vertices.  The emulation runs CTAs
one after another, so this checks the epilogue's arithmetic and the driver's buffers, not their concurrency."""
import pytest

from tests import sweep_drivers as sd
from tests import test_pagerank_row_epilogue_gpu as gpu
from tests.emu_py import surface  # noqa: F401

SCALE = {"f32w": 9, "f64w": 9, "f32": 9}


@pytest.mark.parametrize("etype", list(SCALE))
@pytest.mark.parametrize("layout", list(gpu.LAYOUTS))
def test_pagerank_row_epilogue_emulated(surface, monkeypatch, capfd, layout, etype):  # noqa: F811
    gpu.run_layout(monkeypatch, capfd, gpu.graph_for(etype, SCALE[etype], layout), layout, steps=(1, 2, 5, 10))


@pytest.mark.parametrize("layout", list(gpu.LAYOUTS))
def test_pagerank_row_epilogue_launches_emulated(surface, monkeypatch, capfd, layout):  # noqa: F811
    graph = gpu.graph_for("f32", SCALE["f32"], layout)
    h, g = graph.create(monkeypatch, gpu.LAYOUTS[layout])
    gpu.check_launches(h, g, graph)
    gpu.check_not_converged(h, g, graph)


@pytest.mark.parametrize("T", [sd.np.float32, sd.np.float64])
def test_pagerank_row_epilogue_dangling_emulated(surface, monkeypatch, T):  # noqa: F811
    gpu.test_pagerank_row_epilogue_dangling(monkeypatch, T)
