"""The traversal shape checks of tests/test_traversal_shapes_gpu.py on the CPU emulation of the library
(tests/emu_py.py), at EMU_SIZES: the long path (random and int64 ids), the grid, the lollipop and the brooms at the
single-CTA SSSP limits, every weight family in fp32 and fp64, the exact cutoffs, the BFS depth limits and extract_paths,
against the oracle and against the default run of the same graph."""
import numpy as np
import pytest

from tests import test_traversal_shapes_gpu as shapes
from tests.emu_py import surface  # noqa: F401

SZ = shapes.EMU_SIZES


@pytest.mark.parametrize("shape", ["path-random-ids", "path-int64-ids", "grid", "lollipop", "components", "broom-2048"])
def test_bfs_shapes_emulated(surface, monkeypatch, shape):
    shapes.check_bfs(monkeypatch, shapes.make_shape(shape, SZ))


@pytest.mark.parametrize("shape", ["path", "grid", "lollipop"])
def test_extract_paths_shapes_emulated(surface, monkeypatch, shape):
    shapes.check_extract_paths(monkeypatch, shapes.make_shape(shape, SZ))


@pytest.mark.parametrize("wdtype", [np.float32, np.float64])
@pytest.mark.parametrize("family", shapes.FAMILIES)
def test_sssp_shapes_emulated(surface, monkeypatch, family, wdtype):
    """every weight family and cutoff on the path (symmetric: long zero-weight plateaus) and the grid (every form)"""
    shapes.check_sssp(monkeypatch, shapes.make_shape("path-random-ids", SZ), family, wdtype, knob_sets={},
                      forms=shapes.FORMS[:1])
    shapes.check_sssp(monkeypatch, shapes.make_shape("grid", SZ), family, wdtype, knob_sets={})


@pytest.mark.parametrize("wdtype", [np.float32, np.float64])
def test_sssp_knobs_emulated(surface, monkeypatch, wdtype):
    shapes.check_sssp(monkeypatch, shapes.make_shape("grid", SZ), "zero70", wdtype, cutoffs=False, forms=shapes.FORMS[:1])


@pytest.mark.parametrize("wdtype", [np.float32, np.float64])
def test_sssp_lollipop_int64_ids_emulated(surface, monkeypatch, wdtype):
    for shape, family in (("lollipop", "loguniform"), ("path-int64-ids", "zero70")):
        shapes.check_sssp(monkeypatch, shapes.make_shape(shape, SZ), family, wdtype, knob_sets={}, cutoffs=False)


@pytest.mark.parametrize("shape", ["broom-2048", "broom-2049"])
def test_sssp_broom_emulated(surface, monkeypatch, shape):
    sh = shapes.make_shape(shape, SZ)
    shapes.check_sssp(monkeypatch, sh, "unit", np.float32, knob_sets={}, cutoffs=False)
    shapes.check_sssp(monkeypatch, sh, "ints", np.float64, knob_sets={}, cutoffs=False, forms=shapes.FORMS[:1])
