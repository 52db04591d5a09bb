"""The pull sweep on the H100, row by row against an fp64 reference (tests/sweep_rows.py), on every layout path, tail bound
and element type: the plain sweep with 32- and 64-bit offsets, the piece stream without a tail and with tail bounds 2, 4, 8,
16 and 32, forced bands, and the F slots without bank order.  The block sweep (cugraph_b200_block_pull_sweep) runs the
library's pull_sweep on one GPU with a caller-chosen x, so every row of y can be checked after each of three consecutive
sweeps into the same y with different x and alpha (the tail's work cursor is reset by the previous sweep's last band).

Graphs: the ladder (every in-degree 1..31 in runs whose ends sit at and around tile and work-unit bounds, rotated over
seeds so that at bound 32 every degree meets every run length; more than 2048 hubs, an odd stream row count at bounds 16
and 32 and a variant with a multiple of 512; more than two column blocks of either width), RMAT-16, and tall and wide
rectangular blocks.  The worst |y - y*| / tol per element type and path is printed at the end of the module.

Then one PageRank iteration from an initial guess on RMAT-15 (CSC, and CSR through the re-sorted pull view) against an
fp64 evaluation of the update rule: the init term, empty rows = init and the single-GPU layout built by pull_view."""
import collections

import numpy as np
import pytest

from oracle.rmat import rmat_edgelist
from tests import sweep_rows as sr

pytestmark = pytest.mark.gpu

WORST = collections.defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def report_margins(request):
    """the margins on record: printed past pytest's output capture when the module is done"""
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    if WORST and capman is not None:
        with capman.global_and_fixture_disabled():
            print("\nworst |y - y*| / tol per element type and path:")
            for k in sorted(WORST):
                print(f"  {k:<40} {WORST[k]:.3e}")


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
    if _capi.emulated():                        # emu/run_gpu_suite_on_cpu.py: the emulated device's L2
        return 1 << 20
    return int(torch.cuda.get_device_properties(0).L2_cache_size)


TYPES = {"f32": (np.float32, False), "f32w": (np.float32, True), "f64w": (np.float64, True)}
STREAM = {"SWEEP_MIN_EDGES": 0}
LAYOUTS = {"plain": {}, "plain-offs64": {"OFFS64_MIN_EDGES": 0},
           **{f"tail{b}": {**STREAM, "SWEEP_TAIL_DEGREE": b} for b in (1, 2, 4, 8, 16, 32)},
           "bands3-tail16": {**STREAM, "SWEEP_TAIL_DEGREE": 16, "SWEEP_BANDS": 3},
           "bands5-tail32": {**STREAM, "SWEEP_TAIL_DEGREE": 32, "SWEEP_BANDS": 5},
           "nobank-tail16": {**STREAM, "SWEEP_TAIL_DEGREE": 16, "SWEEP_BANK_ORDER": 0}}
LADDER = [(t, p) for p in LAYOUTS for t in TYPES if not (p.startswith("nobank") and t == "f64w")]


def _run(lib, monkeypatch, capfd, l2, rows, cols, n_rows, n_cols, etype, path, label, wseed=5):
    dtype, weighted = TYPES[etype]
    w = sr.weights(rows.size, dtype, wseed) if weighted else None
    knobs = LAYOUTS[path]
    r = sr.run_block(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2, f"{label} {etype} {path}")
    WORST[f"{etype} {path}"] = max(WORST[f"{etype} {path}"], r)
    return knobs


@pytest.mark.parametrize("etype,path", LADDER, ids=[f"{t}-{p}" for t, p in LADDER])
def test_ladder_rows(lib, l2_bytes, monkeypatch, capfd, etype, path):
    rows, cols, n_rows, n_cols = sr.ladder(seed=0)
    knobs = _run(lib, monkeypatch, capfd, l2_bytes, rows, cols, n_rows, n_cols, etype, path, "ladder")
    bound = knobs.get("SWEEP_TAIL_DEGREE")
    if bound in (16, 32):                       # an odd last stream row: k_sweep_finish's single-row load
        n_str = sr.stream_rows(rows, max(n_rows, n_cols), bound)
        assert n_str % 2 == 1 and n_str % 512 != 0
    if "SWEEP_BANDS" in knobs:                  # the builder may round to fewer bands than asked, but not to one
        assert sr.expected_layout(np.bincount(rows, minlength=n_cols), rows.size, knobs, 4, l2_bytes)["bands"] >= 2


@pytest.mark.parametrize("seed", range(1, 8))
@pytest.mark.parametrize("etype", list(TYPES))
def test_ladder_rotated_runs_bound32(lib, l2_bytes, monkeypatch, capfd, seed, etype):
    """with the seeds of test_ladder_rows, every in-degree 1..31 meets every run length of sr.run_lengths in the tail"""
    rows, cols, n_rows, n_cols = sr.ladder(seed=seed)
    _run(lib, monkeypatch, capfd, l2_bytes, rows, cols, n_rows, n_cols, etype, "tail32", f"ladder seed {seed}", wseed=seed)


@pytest.mark.parametrize("path", ["tail32", "bands5-tail32"])
@pytest.mark.parametrize("etype", list(TYPES))
def test_ladder_stream_rows_multiple_of_512(lib, l2_bytes, monkeypatch, capfd, etype, path):
    rows, cols, n_rows, n_cols = sr.ladder(seed=2, n_hubs=2560)
    assert sr.stream_rows(rows, n_cols, 32) == 2560
    _run(lib, monkeypatch, capfd, l2_bytes, rows, cols, n_rows, n_cols, etype, path, "ladder 5x512")


RMAT_PATHS = [("f32", "plain"), ("f32w", "tail8"), ("f64w", "tail8"), ("f32", "bands3-tail16"), ("f32w", "tail16"),
              ("f64w", "bands3-tail16"), ("f32w", "tail32"), ("f64w", "tail32"), ("f32", "nobank-tail16")]


@pytest.mark.parametrize("etype,path", RMAT_PATHS, ids=[f"{t}-{p}" for t, p in RMAT_PATHS])
def test_rmat16_rows(lib, l2_bytes, monkeypatch, capfd, etype, path):
    s, d = rmat_edgelist(16, 16 << 16, seed=316)
    _run(lib, monkeypatch, capfd, l2_bytes, d, s, 1 << 16, 1 << 16, etype, path, "rmat-16")


RECT = [(shape, t, p) for shape in ("tall", "wide") for t in ("f32w", "f64w") for p in ("tail16", "bands3-tail16", "tail32")]


@pytest.mark.parametrize("shape,etype,path", RECT, ids=[f"{s}-{t}-{p}" for s, t, p in RECT])
def test_rectangular_block_rows(lib, l2_bytes, monkeypatch, capfd, shape, etype, path):
    """tall: the tail's padding column (the span) lies past n_cols; wide: more column blocks than the rows span"""
    n_rows, n_cols = (130_000, 60_000) if shape == "tall" else (40_000, 123_000)
    rows, cols = sr.random_block(n_rows, n_cols, 2100, 9000, seed=41 if shape == "tall" else 42)
    _run(lib, monkeypatch, capfd, l2_bytes, rows, cols, n_rows, n_cols, etype, path, shape)


# ---- one PageRank iteration through the single-GPU graph path
PR_KNOBS = {"tail2": {**STREAM, "SWEEP_TAIL_DEGREE": 2}, "tail16": {**STREAM, "SWEEP_TAIL_DEGREE": 16},
            "tail32": {**STREAM, "SWEEP_TAIL_DEGREE": 32}, "bands3": {**STREAM, "SWEEP_BANDS": 3}}


@pytest.mark.parametrize("knob", list(PR_KNOBS))
@pytest.mark.parametrize("store_transposed", [True, False], ids=["csc", "csr"])
@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32w", "f64w"])
def test_pagerank_one_step_rows(l2_bytes, monkeypatch, capfd, knob, store_transposed, wdtype):
    import torch
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import make_graph
    knobs = PR_KNOBS[knob]
    for k in sr.KNOBS:
        monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)
    for k, v in knobs.items():
        monkeypatch.setenv("CUGRAPH_B200_" + k, str(v))
    monkeypatch.setenv("CUGRAPH_B200_BUILD_TRACE", "1")
    scale, alpha = 15, 0.85
    V = 1 << scale
    s, d = rmat_edgelist(scale, 16 << scale, seed=415)
    w = sr.weights(s.size, wdtype, 11)
    capfd.readouterr()
    h, g = make_graph(s, d, w, store_transposed=store_transposed, weight_dtype=wdtype, vertices=np.arange(V, dtype=np.int32))
    v0, p0, _ = plc.pagerank(h, g, None, None, None, None, alpha, 0.0, 3, False, fail_on_nonconvergence=False)
    v1, p1, _ = plc.pagerank(h, g, None, None, v0, p0, alpha, 0.0, 1, False, fail_on_nonconvergence=False)
    es = np.dtype(wdtype).itemsize
    sr.check_trace(capfd.readouterr().err, sr.expected_layout(np.bincount(d, minlength=V), s.size, knobs, es, l2_bytes),
                   f"pagerank {knob}")
    assert torch.equal(v0, v1) and p1.dtype == (torch.float64 if es == 8 else torch.float32)
    vv = v0.cpu().numpy()
    pos = np.empty(V, np.int64)
    pos[vv] = np.arange(V)
    q = p0.cpu().numpy().astype(np.float64)
    q = q / q.sum()                                           # the driver normalises an initial guess
    outw = np.bincount(pos[s], weights=w.astype(np.float64), minlength=V)
    x = np.where(outw > 0, q / np.where(outw > 0, outw, 1.0), 0.0)
    y = np.bincount(pos[d], weights=x[pos[s]] * w.astype(np.float64), minlength=V)
    ref = alpha * y + (alpha * q[outw == 0].sum() + 1.0 - alpha) / V
    got = p1.cpu().numpy().astype(np.float64)
    indeg = np.bincount(pos[d], minlength=V)
    assert (indeg == 0).sum() > 1000                          # empty rows = the init term, checked with the rest
    rel = np.abs(got - ref) / ref
    tol = 1e-12 if es == 8 else 1e-6
    r = int(np.argmax(rel))
    assert rel[r] < tol, f"vertex {r} (in-degree {int(indeg[r])}): got {got[r]!r}, expected {ref[r]!r}, rel {rel[r]:.3g}"
    WORST[f"pagerank {'f64w' if es == 8 else 'f32w'} {knob} (rel / tol)"] = max(
        WORST[f"pagerank {'f64w' if es == 8 else 'f32w'} {knob} (rel / tol)"], float(rel[r]) / tol)
