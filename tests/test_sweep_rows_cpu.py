"""The row-by-row sweep checks of tests/sweep_rows.py on the CPU, over the emulation build of the library (tests/emu_py.py):
the ladder (more than two column blocks of either element width, every tail degree, run ends around tile and work-unit
bounds), one RMAT-12 block and the tall block, under a reduced set of knobs that still has tail bounds 16 and 32, forced
bands and fp64.  The emulation runs CTAs one after another, so this checks the layout and the kernels' logic, not their
concurrency."""
import numpy as np
import pytest

from oracle.rmat import rmat_edgelist
from tests import sweep_rows as sr

EMU_L2 = 1 << 20          # the emulated device's L2 (emu/cuda_runtime.h)


@pytest.fixture(scope="module")
def lib():
    pytest.importorskip("torch")
    from tests.emu_py import emulated_python_surface
    try:
        cm = emulated_python_surface()
        L = cm.__enter__()
    except Exception as e:  # no host compiler
        pytest.skip(f"emulation build unavailable: {e}")
    yield L
    cm.__exit__(None, None, None)


TYPES = {"f32": (np.float32, False), "f32w": (np.float32, True), "f64w": (np.float64, True)}
LADDER = [("f32", "plain", {}), ("f64w", "plain-offs64", {"OFFS64_MIN_EDGES": 0}),
          ("f32w", "no-tail", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 1}),
          ("f32", "tail16", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}),
          ("f64w", "tail16", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}),
          ("f32w", "tail32", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 32}),
          ("f64w", "bands5-tail32", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 32, "SWEEP_BANDS": 5}),
          ("f32", "bands3-tail16-nobank", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16, "SWEEP_BANDS": 3,
                                           "SWEEP_BANK_ORDER": 0})]


@pytest.mark.parametrize("etype,path,knobs", LADDER, ids=[f"{e}-{p}" for e, p, _ in LADDER])
def test_ladder_rows_emulated(lib, monkeypatch, capfd, etype, path, knobs):
    dtype, weighted = TYPES[etype]
    rows, cols, n_rows, n_cols = sr.ladder(seed=3)
    w = sr.weights(rows.size, dtype, 5) if weighted else None
    sr.run_block(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, EMU_L2, f"ladder {etype} {path}")


@pytest.mark.parametrize("etype,knobs", [("f32w", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 8}),
                                         ("f64w", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 32, "SWEEP_BANDS": 2})])
def test_rmat12_rows_emulated(lib, monkeypatch, capfd, etype, knobs):
    dtype, weighted = TYPES[etype]
    s, d = rmat_edgelist(12, 16 << 12, seed=12)
    w = sr.weights(s.size, dtype, 6) if weighted else None
    sr.run_block(lib, monkeypatch, capfd, d, s, w, 1 << 12, 1 << 12, dtype, knobs, EMU_L2, f"rmat-12 {etype}")


def test_tall_block_rows_emulated(lib, monkeypatch, capfd):
    """n_rows > n_cols: the tail's padding column (the span) lies past the last column"""
    rows, cols = sr.random_block(110_000, 60_000, 700, 4000, seed=21)
    w = sr.weights(rows.size, np.float64, 7)
    sr.run_block(lib, monkeypatch, capfd, rows, cols, w, 110_000, 60_000, np.float64,
                 {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 32, "SWEEP_BANDS": 2}, EMU_L2, "tall f64w")
