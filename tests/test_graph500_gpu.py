"""Generator slices, the BFS / SSSP certificate and the Graph500 harness on the GPU.

- Slices at RMAT-20: mg.rmat_edgelist_share, the _at entry points and pylibcugraph.generate_rmat_edgelist(multi_gpu=True)
  concatenate to the one-call output and to the numpy twin, bit for bit.
- The certificate accepts MGGraph.bfs / sssp results on grids 1x1, 1x2, 2x1, 2x2 and 4x2 of one GPU (tests/mg_world.py) on
  RMAT-16, the forced-predecessor graph, the zero-weight graph and isolated vertices, and single-GPU cugraph_bfs /
  cugraph_sssp results on a 1x1 grid; it rejects the corruptions with the counter named for each.
- The harness driver at scale 16 with 4 roots on grids 1x1, 2x2 and 4x2: every root validated, the same distances and
  edges_from_reached on every grid; and end to end in a world-size-1 NCCL group with single_gpu."""
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import graph500_ref as ref  # noqa: E402
from tests import mg_procs, mg_sssp_ref, mg_world  # noqa: E402

pytestmark = pytest.mark.gpu

GRIDS = [(1, 1), (1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x1", "1x2", "2x1", "2x2", "4x2"]


def _world(monkeypatch, R, Cc):
    return mg_world.grid_world(monkeypatch, R, Cc) if R * Cc > 1 else 1


def _mirror_worker(rank, world, scale, counts, seed):
    from cugraph_b200 import pylibcugraph as plc
    out = plc.generate_rmat_edgelist(plc.ResourceHandle(), seed, scale, counts[rank], 0.57, 0.19, 0.19, False, True, True,
                                     0.0, 1.0, np.float32, True, True, 0, 4, multi_gpu=True)
    return [None if x is None else x.cpu().numpy() for x in out]


@pytest.mark.parametrize("P", [1, 3, 8])
def test_slices_rmat20(P):
    from oracle.rmat import rmat_edgelist_counter, uniform_counter
    from cugraph_b200 import mg
    from cugraph_b200 import pylibcugraph as plc
    from cugraph_b200.generators import rmat_edgelist, uniform_values
    import torch
    scale, E, seed = 20, (1 << 20) + 5, 0
    one_s, one_d = rmat_edgelist(scale, E, seed=seed)
    rs, rd = rmat_edgelist_counter(scale, E, seed=seed)
    assert np.array_equal(one_s.cpu().numpy(), rs) and np.array_equal(one_d.cpu().numpy(), rd)
    ss, dd, ww = [], [], []
    for r in range(P):
        s, d, first = mg.rmat_edgelist_share(scale, E, seed=seed, groups=mg.Groups(P, r, P, 1, r, 0, None, None))
        ss.append(s)
        dd.append(d)
        ww.append(uniform_values(s.numel(), 2, 0.0, 1.0, torch.float32, first=first))
    assert torch.equal(torch.cat(ss), one_s) and torch.equal(torch.cat(dd), one_d)
    assert np.array_equal(torch.cat(ww).cpu().numpy(), uniform_counter(E, 2, 0.0, 1.0, np.float32))
    counts = [E // P + (r % 2) for r in range(P)]
    res = mg_world.run(P, _mirror_worker, scale, counts, seed)
    single = plc.generate_rmat_edgelist(plc.ResourceHandle(), seed, scale, sum(counts), 0.57, 0.19, 0.19, False, True, True,
                                        0.0, 1.0, np.float32, True, True, 0, 4, multi_gpu=False)
    for k in range(5):
        assert np.array_equal(np.concatenate([r[k] for r in res]), single[k].cpu().numpy()), k


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_certificate_accepts_on_one_gpu(monkeypatch, R, Cc):
    world = _world(monkeypatch, R, Cc)
    for wdtype in (np.float32, np.float64):
        s, d, w, V = mg_sssp_ref.rmat_graph(16, wdtype)
        runs = ref.rmat_runs(s, V)
        if wdtype == np.float64:
            runs = [r for r in runs if r[0] == "sssp"]
        for run, (cert, _) in zip(runs, ref.accept(s, d, w, world, runs, device="cuda")):
            ref.assert_accepts(cert, run)
    s, d, runs = ref.forced()
    for run, (cert, _) in zip(runs, ref.accept(s, d, None, world, runs, device="cuda")):
        ref.assert_accepts(cert, run)
    for wdtype in (np.float32, np.float64):
        s, d, w, V = mg_sssp_ref.zero_weight_graph(wdtype)
        runs = [("sssp", 0, {}), ("sssp", 7, {})]
        for run, (cert, _) in zip(runs, ref.accept(s, d, w, world, runs, device="cuda")):
            ref.assert_accepts(cert, run)
    s, d, w, V = mg_sssp_ref.rmat_graph(12, np.float32)
    runs = [("bfs", int(s[0]), {}), ("sssp", int(s[0]), {})]
    for run, (cert, _) in zip(runs, ref.accept(s, d, w, world, runs, vertices=np.arange(V, V + 37, dtype=np.int32),
                                               device="cuda")):
        ref.assert_accepts(cert, run)


def test_certificate_single_gpu_results_on_one_gpu():
    s, d, w, V = mg_sssp_ref.rmat_graph(16, np.float32)
    c_bfs, c_sssp, c_bad = ref.single_gpu_certificates(s, d, w, V, int(s[0]), device="cuda")
    ref.assert_accepts(c_bfs, "bfs")
    ref.assert_accepts(c_sssp, "sssp")
    assert not c_bad["ok"] and c_bad["root"] == 1


def test_certificate_rejects_on_one_gpu(monkeypatch):
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, w, V = mg_sssp_ref.rmat_graph(12, np.float32)
    source = mg_sssp_ref.sources(s, V)[0]
    run = ("bfs", source, {})
    (cert, parts), = ref.accept(s, d, None, world, [run], device="cuda")
    ref.assert_accepts(cert, run)
    cases = ref.bfs_corruptions(s, d, parts, source)
    for (rule, _), c in zip(cases, ref.reject(s, d, None, world, run, parts, [ref.edit(parts, fn) for _, fn in cases],
                                              device="cuda")):
        assert not c["ok"] and c[rule] > 0, (rule, c)
    s, d, w, V = mg_sssp_ref.zero_weight_graph(np.float32)
    run = ("sssp", 0, {})
    (cert, parts), = ref.accept(s, d, w, world, [run], device="cuda")
    ref.assert_accepts(cert, run)
    res = ref.by_id(parts)
    v = next(x for x, (dv, p) in res.items() if p >= 0 and dv > 0)
    edits = [ref.edit(parts, ref.set_at(v, dist=np.nan)), ref.edit(parts, ref.zero_cycle(s, d, w, parts, 0))]
    c_nan, c_cycle = ref.reject(s, d, w, world, run, parts, edits, device="cuda")
    assert not c_nan["ok"] and c_nan["bad_value"] > 0
    assert not c_cycle["ok"] and c_cycle["cycle"] >= 2 and c_cycle["tree_edge"] == 0


# ------------------------------------------------------------------------------------------------------------ harness
def _harness_worker(rank, world):
    from cugraph_b200 import mg
    from scripts.graph500 import run
    return run(mg.make_groups(), 16, n_roots=4, keep_results=True)


def test_harness_world_size_independent(monkeypatch):
    got = {}
    for R, Cc in ((1, 1), (2, 2), (4, 2)):
        world = _world(monkeypatch, R, Cc)
        res = mg_world.run(world, _harness_worker)
        out = res[0]
        assert out["ok"] and out["grid"] == f"{R}x{Cc}"
        for k in ("bfs", "sssp"):
            assert out[k]["validated"] == out[k]["roots"] == 4
        per = {}
        for k in ("bfs", "sssp"):
            runs = []
            for i in range(4):
                parts = [(r["results"][k][i][0], r["results"][k][i][1]) for r in res]
                fill, dt = (ref.IMAX, np.int32) if k == "bfs" else (np.finfo(np.float32).max, np.float32)
                runs.append((mg_world.by_id(parts, 1 << 16, fill, dt), res[0]["results"][k][i][2]))
            per[k] = runs
        got[(R, Cc)] = (out["bfs"]["roots"], per)
    base = got[(1, 1)][1]
    for key, (_, per) in got.items():
        for k in ("bfs", "sssp"):
            for (d0, e0), (d1, e1) in zip(base[k], per[k]):
                assert e0 == e1, (key, k)
                assert np.array_equal(d0, d1), (key, k)


def _nccl_worker(rank, world):
    from cugraph_b200 import mg
    from scripts.graph500 import run
    return run(mg.make_groups(), 16, n_roots=8, single_gpu=True)


def test_harness_nccl_world_size_1_single_gpu():
    out, = mg_procs.run(_nccl_worker, 1, backend="nccl", timeout=900)
    assert out["ok"] and out["grid"] == "1x1" and out["roots"] == 8
    for kern in (out["bfs"], out["sssp"], out["single_gpu"]["bfs"], out["single_gpu"]["sssp"]):
        assert kern["validated"] == kern["roots"] == 8
        assert set(kern["time_s"]) == {"min", "q1", "median", "q3", "max", "mean", "stddev"}
        assert {"harmonic_mean", "harmonic_stddev"} <= set(kern["teps"])
        assert kern["validation_s_per_root"] > 0
    for key in ("scale", "edge_factor", "grid", "n_gpus", "roots", "construction_s", "direction_optimizing", "root_rule",
                "timing"):
        assert key in out
