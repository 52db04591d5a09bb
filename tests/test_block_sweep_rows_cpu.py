"""The block sweep in both orientations (tests/block_sweep_rows.py) on the CPU, over the emulation build of the library
(tests/emu_py.py): the transposed sweep on the plain sweep with 32- and 64-bit offsets and on the piece stream with tail
bounds 1 / 16 / 32 and forced bands, for float32, weighted float32 and float64 blocks, with and without the weights; pull and
transposed sweeps of one block interleaved into two y arrays; a transposed sweep after SSSP or WCC built the column-major
copy; transposed = FALSE against cugraph_b200_block_pull_sweep; the entry point's error paths."""
import ctypes as C

import numpy as np
import pytest

from tests import block_sweep_rows as bsr
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
CASES = [("f32", "plain", {}, True), ("f64w", "plain-offs64", {"OFFS64_MIN_EDGES": 0}, True),
         ("f32w", "no-tail", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 1}, True),
         ("f32w", "no-tail-unweighted", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 1}, False),
         ("f32", "tail16", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}, True),
         ("f64w", "tail16-unweighted", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}, False),
         ("f64w", "bands3-tail32", {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 32, "SWEEP_BANDS": 3}, True)]


def _ladder_t(seed=3):
    """the ladder of tests/sweep_rows.py with rows and columns exchanged: its transpose is the ladder (every tail degree,
    more than two column blocks of either width)"""
    rows, cols, n_rows, n_cols = sr.ladder(seed=seed)
    return cols, rows, n_cols, n_rows


@pytest.mark.parametrize("etype,path,knobs,use_weights", CASES, ids=[f"{e}-{p}" for e, p, _, _ in CASES])
def test_transposed_rows_emulated(lib, monkeypatch, capfd, etype, path, knobs, use_weights):
    dtype, weighted = TYPES[etype]
    rows, cols, n_rows, n_cols = _ladder_t()
    w = sr.weights(rows.size, dtype, 5) if weighted else None
    bsr.run(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, EMU_L2, f"ladder^T {etype} {path}",
            use_weights=use_weights)


@pytest.mark.parametrize("knobs", [{}, {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}], ids=["plain", "tail16"])
def test_pull_and_transposed_interleaved_emulated(lib, monkeypatch, capfd, knobs):
    rows, cols = sr.random_block(30_000, 50_000, 300, 3000, seed=31)
    w = sr.weights(rows.size, np.float32, 8)
    bsr.run(lib, monkeypatch, capfd, rows, cols, w, 30_000, 50_000, np.float32, knobs, EMU_L2, "interleaved", interleave=True)


@pytest.mark.parametrize("first", ["wcc", "sssp"])
def test_transposed_after_push_copy_emulated(lib, monkeypatch, capfd, first):
    rows, cols = sr.random_block(20_000, 20_000, 200, 2000, seed=41)
    w = sr.weights(rows.size, np.float64, 9)
    bsr.run(lib, monkeypatch, capfd, rows, cols, w, 20_000, 20_000, np.float64,
            {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 32}, EMU_L2, f"after {first}", first=first)


def test_untransposed_sweep_is_pull_sweep_emulated(lib, monkeypatch, capfd):
    rows, cols = sr.random_block(20_000, 30_000, 200, 2000, seed=51)
    w = sr.weights(rows.size, np.float32, 10)
    bsr.pull_entries_agree(lib, monkeypatch, capfd, rows, cols, w, 20_000, 30_000, np.float32,
                           {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}, EMU_L2, "pull entries")


def test_block_sweep_errors_emulated(lib):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    handle = ResourceHandle(stream=0)
    keep = [torch.tensor([0, 1, 2], dtype=torch.int32), torch.tensor([1, 2, 0], dtype=torch.int32),
            torch.tensor([0.5, 0.25, 1.0])]
    vs = [View(k) for k in keep]
    blk, err = C.c_void_p(), C.c_void_p()
    _capi.check(lib.cugraph_b200_block_create(handle.ptr, 3, 4, vs[0].ptr, vs[1].ptr, vs[2].ptr, C.byref(blk), C.byref(err)),
                err, "cugraph_b200_block_create")
    span = int(lib.cugraph_b200_block_span(blk.value))
    n_x = int(lib.cugraph_b200_padded_elems(span, 4))
    x, y = torch.zeros(n_x), torch.zeros(span)
    x[:3] = torch.tensor([1.0, 2.0, 4.0])

    def sweep(xx, yy, transposed=1, use_weights=1, b=blk.value):
        vx, vy = View(xx), View(yy)
        e = C.c_void_p()
        code = lib.cugraph_b200_block_sweep(handle.ptr, b, transposed, use_weights, vx.ptr, vy.ptr, 1.0, C.byref(e))
        vx.free()
        vy.free()
        _capi.check(code, e, "cugraph_b200_block_sweep")

    sweep(x, y)                                  # edges (0,1) (1,2) (2,0): y[col] = x[row] * w
    assert y.tolist()[:3] == [4.0, 0.5, 0.5]
    sweep(x, y, use_weights=0)
    assert y.tolist()[:3] == [4.0, 1.0, 2.0]
    for xx, yy in ((x.double(), y), (x, y.double()), (x[:n_x - 1], y), (x, y[:span - 1])):
        with pytest.raises(_capi.CugraphError) as e:
            sweep(xx, yy)
        assert e.value.code == _capi.INVALID_INPUT
    both = torch.zeros(n_x + span)
    with pytest.raises(_capi.CugraphError) as e:     # x and y overlap
        sweep(both[:n_x], both[n_x - 1:n_x - 1 + span])
    assert e.value.code == _capi.INVALID_INPUT
    with pytest.raises(_capi.CugraphError) as e:
        sweep(x, y, b=None)
    assert e.value.code == _capi.INVALID_INPUT
    lib.cugraph_b200_block_free(blk.value)
    for v in vs:
        v.free()
