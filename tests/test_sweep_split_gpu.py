"""The pull sweep with its tail beside the piece stream (CUGRAPH_B200_SWEEP_TAIL_SMS) on the H100: k_sweep_tail on a share
of the SMs, launched on the handle's side stream, while the bands' k_sweep runs on the others, the two joined before
anything that reads their rows.  Checked against the fp64 restatements at the extremes of the split (the tail on one SM;
the stream on one CTA, the tail on every other SM), in between, and with no split at all; with forced bands, so that a
band's finish runs while the tail does; float32 and float64, weighted and unweighted:

- row by row (tests/sweep_rows.py), three sweeps into the same y one after the other: each tail launch takes the cursor
  slot the one before it left behind;
- PageRank with its row epilogue for 1, 2, 5 and 30 steps (tests/test_pagerank_row_epilogue_gpu.py), and Katz,
  eigenvector, HITS and personalized PageRank step by step (tests/sweep_drivers.py): the dangling and difference sums the
  tail adds into the loop state are complete when the next step reads them;
- one graph through many calls of every driver;
- the launches per iteration: the same with and without the split."""
import numpy as np
import pytest

from tests import sweep_drivers as sd
from tests import sweep_rows as sr
from tests import test_pagerank_row_epilogue_gpu as epi

pytestmark = pytest.mark.gpu

TAIL16 = {"SWEEP_MIN_EDGES": 0, "SWEEP_TAIL_DEGREE": 16}
BANDS = {"SWEEP_MIN_EDGES": 0, "SWEEP_BANDS": 3, "SWEEP_TAIL_DEGREE": 8}
ALL_BUT_ONE = 1 << 20   # clamped to the SM count - 1: the stream on one CTA
SPLITS = {"tail1": {**TAIL16, "SWEEP_TAIL_SMS": 1},
          "stream1": {**TAIL16, "SWEEP_TAIL_SMS": ALL_BUT_ONE},
          "tail32": {**TAIL16, "SWEEP_TAIL_SMS": 32},
          "serial": {**TAIL16, "SWEEP_TAIL_SMS": 0},
          "default": TAIL16,
          "bands-tail1": {**BANDS, "SWEEP_TAIL_SMS": 1},
          "bands-tail40": {**BANDS, "SWEEP_TAIL_SMS": 40},
          "bands-stream1": {**BANDS, "SWEEP_TAIL_SMS": ALL_BUT_ONE}}
TYPES = {"f32": (np.float32, False), "f32w": (np.float32, True), "f64w": (np.float64, True)}
SCALE = {"f32w": 16, "f64w": 15, "f32": 16}


@pytest.fixture(scope="module")
def lib():
    import torch
    from cugraph_b200 import _capi
    torch.cuda.set_device(0)
    return _capi.lib()


@pytest.fixture(scope="module")
def l2_bytes():
    import torch
    return int(torch.cuda.get_device_properties(0).L2_cache_size)


def _split_trace(err):
    """(tail SMs, SMs) of every split line of the build trace"""
    import re
    return [tuple(map(int, m)) for m in re.findall(r"\[sweep\] split: tail on (\d+) of (\d+) SMs", err)]


@pytest.mark.parametrize("etype", list(TYPES))
@pytest.mark.parametrize("split", list(SPLITS))
def test_split_rows(lib, l2_bytes, monkeypatch, capfd, split, etype):
    dtype, weighted = TYPES[etype]
    rows, cols, n_rows, n_cols = sr.ladder(seed=1)
    w = sr.weights(rows.size, dtype, 5) if weighted else None
    monkeypatch.delenv("CUGRAPH_B200_SWEEP_TAIL_SMS", raising=False)
    knobs = SPLITS[split]
    capfd.readouterr()
    # run_block checks the layout against the build trace and consumes it: the split line is checked in the next test
    sr.run_block(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, f"ladder {etype} {split}")


@pytest.mark.parametrize("split", list(SPLITS))
def test_split_trace(monkeypatch, capfd, split):
    """the build trace names the split; a forced value is clamped to [0, SMs - 1]"""
    import torch
    graph = sd.graph_of("f32w", SCALE["f32w"])
    capfd.readouterr()
    h, g = graph.create(monkeypatch, SPLITS[split])
    sd.check_pagerank(h, g, graph, steps=3)   # builds the layout
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = _split_trace(capfd.readouterr().err)
    assert got and all(n == sms for _, n in got), got
    forced = SPLITS[split].get("SWEEP_TAIL_SMS")
    if forced is not None:
        assert all(k == min(forced, sms - 1) for k, _ in got), (split, got)
    else:
        assert all(0 <= k < sms for k, _ in got), got


@pytest.mark.parametrize("etype", list(TYPES))
@pytest.mark.parametrize("split", ["bands-tail1", "stream1", "tail32"])
def test_split_pagerank(monkeypatch, capfd, split, etype):
    monkeypatch.setitem(epi.LAYOUTS, split, SPLITS[split])
    epi.run_layout(monkeypatch, capfd, epi.graph_for(etype, SCALE[etype], "csc"), split)


@pytest.mark.parametrize("etype", ["f32w", "f64w"])
@pytest.mark.parametrize("split", ["bands-tail40", "stream1"])
@pytest.mark.parametrize("algorithm", ["katz", "eigenvector", "hits", "personalized"])
def test_split_drivers(monkeypatch, capfd, algorithm, split, etype):
    monkeypatch.setitem(sd.KNOBS, split, SPLITS[split])
    sd.run_case(algorithm, monkeypatch, capfd, sd.graph_of(etype, SCALE[etype]), split)


@pytest.mark.parametrize("split", ["tail1", "bands-stream1"])
def test_split_many_calls(monkeypatch, capfd, split):
    monkeypatch.setitem(sd.KNOBS, split, SPLITS[split])
    sd.run_many_calls(monkeypatch, capfd, sd.graph_of("f32w", SCALE["f32w"]), split)


def test_split_launches(monkeypatch, capfd):
    """a PageRank iteration launches as many kernels with the tail beside the stream as after it (the side stream's
    launch counts like any other), two fewer than a personalized one"""
    graph = sd.graph_of("f32", SCALE["f32"])
    per_iteration = {}
    for split in ("serial", "tail32", "bands-tail1", "bands-stream1"):
        h, g = graph.create(monkeypatch, SPLITS[split])
        epi.check_launches(h, g, graph)
        counts = []
        for k in (3, 4):
            l0 = h.launch_count()
            sd.pagerank_call(h, g, graph, 0.85, 0.0, k)
            counts.append(h.launch_count() - l0)
        per_iteration[split] = counts[1] - counts[0]
    assert per_iteration["serial"] == per_iteration["tail32"], per_iteration
    assert per_iteration["bands-tail1"] == per_iteration["bands-stream1"], per_iteration
