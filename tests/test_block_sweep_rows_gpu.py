"""The block sweep in both orientations (tests/block_sweep_rows.py) on the GPU: the transposed sweep on the plain sweep with 32-
and 64-bit offsets and on the piece stream with tail bounds 1 / 16 / 32 and forced bands, float32 / weighted float32 /
float64, with and without the weights, on the transposed ladder and on a transposed RMAT-16 block; pull and transposed sweeps
interleaved into two y arrays; a transposed sweep after SSSP or WCC built the column-major copy; transposed = FALSE against
cugraph_b200_block_pull_sweep."""
import numpy as np
import pytest

from oracle.rmat import rmat_edgelist
from tests import block_sweep_rows as bsr
from tests import sweep_rows as sr

pytestmark = pytest.mark.gpu

STREAM = {"SWEEP_MIN_EDGES": 0}
LAYOUTS = {"plain": {}, "plain-offs64": {"OFFS64_MIN_EDGES": 0}, "no-tail": {**STREAM, "SWEEP_TAIL_DEGREE": 1},
           "tail16": {**STREAM, "SWEEP_TAIL_DEGREE": 16}, "tail32": {**STREAM, "SWEEP_TAIL_DEGREE": 32},
           "bands3-tail16": {**STREAM, "SWEEP_TAIL_DEGREE": 16, "SWEEP_BANDS": 3}}
TYPES = {"f32": (np.float32, False), "f32w": (np.float32, True), "f64w": (np.float64, True)}
CASES = [(t, p, uw) for t in TYPES for p in LAYOUTS for uw in ((True, False) if TYPES[t][1] else (True,))]


@pytest.fixture(scope="module")
def lib():
    import torch
    from cugraph_b200 import _capi
    torch.cuda.set_device(0)
    return _capi.lib()


@pytest.fixture(scope="module")
def l2_bytes():
    import torch
    from cugraph_b200 import _capi
    if _capi.emulated():
        return 1 << 20
    return int(torch.cuda.get_device_properties(0).L2_cache_size)


@pytest.mark.parametrize("etype,path,use_weights", CASES, ids=[f"{t}-{p}-{'w' if uw else 'plain'}" for t, p, uw in CASES])
def test_transposed_ladder_rows(lib, l2_bytes, monkeypatch, capfd, etype, path, use_weights):
    dtype, weighted = TYPES[etype]
    rows, cols, n_rows, n_cols = sr.ladder(seed=0)
    w = sr.weights(rows.size, dtype, 5) if weighted else None
    bsr.run(lib, monkeypatch, capfd, cols, rows, w, n_cols, n_rows, dtype, LAYOUTS[path], l2_bytes,
            f"ladder^T {etype} {path}", use_weights=use_weights)


@pytest.mark.parametrize("etype,path", [("f32", "tail16"), ("f64w", "bands3-tail16"), ("f32w", "plain")])
def test_transposed_rmat16_rows(lib, l2_bytes, monkeypatch, capfd, etype, path):
    dtype, weighted = TYPES[etype]
    s, d = rmat_edgelist(16, 16 << 16, seed=316)
    w = sr.weights(s.size, dtype, 6) if weighted else None
    bsr.run(lib, monkeypatch, capfd, d, s, w, 1 << 16, 1 << 16, dtype, LAYOUTS[path], l2_bytes, f"rmat-16^T {etype} {path}")


@pytest.mark.parametrize("path", ["plain", "tail16"])
def test_pull_and_transposed_interleaved(lib, l2_bytes, monkeypatch, capfd, path):
    rows, cols = sr.random_block(40_000, 123_000, 2100, 9000, seed=42)
    w = sr.weights(rows.size, np.float32, 8)
    bsr.run(lib, monkeypatch, capfd, rows, cols, w, 40_000, 123_000, np.float32, LAYOUTS[path], l2_bytes, "interleaved",
            interleave=True)


@pytest.mark.parametrize("first", ["wcc", "sssp"])
def test_transposed_after_push_copy(lib, l2_bytes, monkeypatch, capfd, first):
    rows, cols = sr.random_block(130_000, 60_000, 2100, 9000, seed=41)
    w = sr.weights(rows.size, np.float64, 9)
    bsr.run(lib, monkeypatch, capfd, rows, cols, w, 130_000, 60_000, np.float64, LAYOUTS["tail32"], l2_bytes,
            f"after {first}", first=first)


def test_untransposed_sweep_is_pull_sweep(lib, l2_bytes, monkeypatch, capfd):
    rows, cols = sr.random_block(40_000, 123_000, 2100, 9000, seed=43)
    w = sr.weights(rows.size, np.float32, 10)
    bsr.pull_entries_agree(lib, monkeypatch, capfd, rows, cols, w, 40_000, 123_000, np.float32, LAYOUTS["tail16"], l2_bytes,
                           "pull entries")
