"""Generator slices, the BFS / SSSP certificate and the Graph500 harness on the CPU, over the emulated library
(tests/emu_py.py).

- Slices: per-rank slices of the RMAT and uniform streams (cugraph_b200_generate_*_at through generators.py,
  mg.rmat_edgelist_share, pylibcugraph.generate_rmat_edgelist(multi_gpu=True) on every rank of a one-process world)
  concatenate to the one-call output and to the numpy twin, bit for bit, for counts that do not divide by P.
- The certificate accepts (every counter 0) MGGraph.bfs / sssp results on grids 1x1, 1x2, 2x1, 2x2 and 4x2 on RMAT-10,
  the forced-predecessor graph, the zero-weight graph and a graph with isolated vertices, and single-GPU results given on
  the one rank of a 1x1 grid; it rejects every corruption of a valid result with the counter named for it.
- The harness driver at scale 8 in a world-size-2 gloo group."""
import math
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.rmat import rmat_edgelist_counter, uniform_counter  # noqa: E402
from tests import graph500_ref as ref  # noqa: E402
from tests import mg_procs, mg_sssp_ref, mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 1), (1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x1", "1x2", "2x1", "2x2", "4x2"]


# ---------------------------------------------------------------------------------------------------------- slices
def _mirror_worker(rank, world, scale, counts, seed):
    import torch  # noqa: F401
    from cugraph_b200 import pylibcugraph as plc
    h = plc.ResourceHandle()
    out = plc.generate_rmat_edgelist(h, seed, scale, counts[rank], 0.57, 0.19, 0.19, False, True, True, 0.0, 1.0,
                                     np.float32, True, True, 0, 4, multi_gpu=True)
    return [None if x is None else x.cpu().numpy() for x in out]


@pytest.mark.parametrize("P,scale,E", [(1, 10, 1000), (3, 10, 1001), (4, 12, 4099), (7, 9, 50), (5, 31, 333)])
def test_slices_concatenate_to_one_call(surface, P, scale, E):  # noqa: F811
    import torch
    from cugraph_b200 import mg
    from cugraph_b200 import pylibcugraph as plc
    from cugraph_b200.generators import rmat_edgelist, uniform_values
    seed = 4242
    rs, rd = rmat_edgelist_counter(scale, E, seed=seed)
    one_s, one_d = rmat_edgelist(scale, E, seed=seed)
    assert np.array_equal(one_s.numpy(), rs) and np.array_equal(one_d.numpy(), rd)
    parts, firsts = [], []
    for r in range(P):
        g = mg.Groups(P, r, P, 1, r, 0, None, None)
        s, d, first = mg.rmat_edgelist_share(scale, E, seed=seed, groups=g)
        assert first == r * E // P and s.numel() == (r + 1) * E // P - first
        parts.append((s.numpy(), d.numpy()))
        firsts.append(first)
    assert np.array_equal(np.concatenate([p[0] for p in parts]), rs)
    assert np.array_equal(np.concatenate([p[1] for p in parts]), rd)
    for dtype, tdt in ((np.float32, torch.float32), (np.float64, torch.float64), (np.int32, torch.int32)):
        lo, hi = (0, 9) if dtype == np.int32 else (-1.5, 2.0)
        got = np.concatenate([uniform_values(len(p[0]), seed, lo, hi, tdt, first=f).numpy() for p, f in zip(parts, firsts)])
        assert np.array_equal(got, uniform_counter(E, seed, lo, hi, dtype))
    # the mirror's multi_gpu=True over uneven per-rank counts (one of them 0) against its one call over the total
    counts = [(E * (r + 1) * 7) % (E + 3) // P for r in range(P)]
    counts[-1] = 0 if P > 1 else counts[-1]
    total = sum(counts)
    h = plc.ResourceHandle()
    single = plc.generate_rmat_edgelist(h, seed, scale, total, 0.57, 0.19, 0.19, False, True, True, 0.0, 1.0, np.float32,
                                        True, True, 0, 4, multi_gpu=False)
    res = mg_world.run(P, _mirror_worker, scale, counts, seed)
    for k in range(5):
        cat = np.concatenate([r[k] for r in res])
        assert np.array_equal(cat, single[k].numpy()), k
    ws, wd = rmat_edgelist_counter(scale, total, seed=seed)
    assert np.array_equal(single[0].numpy(), ws) and np.array_equal(single[1].numpy(), wd)
    assert np.array_equal(single[2].numpy(), uniform_counter(total, seed + 0x9E37, 0.0, 1.0, np.float32))
    assert np.array_equal(single[3].numpy(), np.arange(total))


# ---------------------------------------------------------------------------------------------------------- accepts
@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_certificate_accepts_rmat(surface, monkeypatch, R, Cc, wdtype):  # noqa: F811
    world = mg_world.grid_world(monkeypatch, R, Cc) if R * Cc > 1 else 1
    s, d, w, V = mg_sssp_ref.rmat_graph(10, wdtype)
    runs = ref.rmat_runs(s, V)
    if wdtype == np.float64:
        runs = [r for r in runs if r[0] == "sssp"]
    for run, (cert, _) in zip(runs, ref.accept(s, d, w, world, runs)):
        ref.assert_accepts(cert, run)


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_certificate_accepts_forced_zero_weight_and_isolated(surface, monkeypatch, R, Cc):  # noqa: F811
    world = mg_world.grid_world(monkeypatch, R, Cc) if R * Cc > 1 else 1
    s, d, runs = ref.forced()
    for run, (cert, _) in zip(runs, ref.accept(s, d, None, world, runs)):
        ref.assert_accepts(cert, run)
    for wdtype in (np.float32, np.float64):
        s, d, w, V = mg_sssp_ref.zero_weight_graph(wdtype)
        runs = [("sssp", 0, {}), ("sssp", 7, {}), ("bfs", 7, {})]
        for run, (cert, _) in zip(runs, ref.accept(s, d, w, world, runs)):
            ref.assert_accepts(cert, run)
    # isolated vertices (vertices=): given, unreached, without predecessor
    s, d, w, V = mg_sssp_ref.rmat_graph(8, np.float32)
    extra = np.arange(V, V + 37, dtype=np.int32)
    runs = [("bfs", int(s[0]), {}), ("sssp", int(s[0]), {})]
    for run, (cert, parts) in zip(runs, ref.accept(s, d, w, world, runs, vertices=extra)):
        ref.assert_accepts(cert, run)
        got = ref.by_id([tuple(p) for p in parts])
        assert all(x in got for x in extra.tolist())


def test_certificate_accepts_single_gpu_results(surface):  # noqa: F811
    s, d, w, V = mg_sssp_ref.rmat_graph(9, np.float32)
    c_bfs, c_sssp, c_bad = ref.single_gpu_certificates(s, d, w, V, int(s[0]))
    ref.assert_accepts(c_bfs, "bfs")
    ref.assert_accepts(c_sssp, "sssp")
    assert not c_bad["ok"] and c_bad["root"] == 1


# ---------------------------------------------------------------------------------------------------------- rejects
@pytest.mark.parametrize("R,Cc", [(1, 1), (2, 2)], ids=["1x1", "2x2"])
def test_certificate_rejects_corrupted_bfs(surface, monkeypatch, R, Cc):  # noqa: F811
    world = mg_world.grid_world(monkeypatch, R, Cc) if R * Cc > 1 else 1
    s, d, w, V = mg_sssp_ref.rmat_graph(9, np.float32)
    source = mg_sssp_ref.sources(s, V)[0]
    run = ("bfs", source, {})
    (cert, parts), = ref.accept(s, d, None, world, [run])
    ref.assert_accepts(cert, run)
    cases = ref.bfs_corruptions(s, d, parts, source)
    certs = ref.reject(s, d, None, world, run, parts, [ref.edit(parts, fn) for _, fn in cases])
    for (rule, _), c in zip(cases, certs):
        assert not c["ok"] and c[rule] > 0, (rule, c)


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_certificate_rejects_corrupted_sssp(surface, monkeypatch, wdtype):  # noqa: F811
    world = mg_world.grid_world(monkeypatch, 2, 2)
    s, d, w, V = mg_sssp_ref.zero_weight_graph(wdtype)
    run = ("sssp", 0, {})
    (cert, parts), = ref.accept(s, d, w, world, [run])
    ref.assert_accepts(cert, run)
    res = ref.by_id(parts)
    v = next(x for x, (dv, p) in res.items() if p >= 0 and dv > 0)
    edits = [ref.edit(parts, ref.set_at(v, dist=np.nan)), ref.edit(parts, ref.zero_cycle(s, d, w, parts, 0)),
             ref.edit(parts, ref.set_at(v, dist=res[v][0] * 2 + 1)), ref.edit(parts, ref.set_at(0, pred=v))]
    certs = ref.reject(s, d, w, world, run, parts, edits)
    for rule, c in zip(("bad_value", "cycle", "edge", "root"), certs):
        assert not c["ok"] and c[rule] > 0, (rule, c)
    assert certs[1]["tree_edge"] == 0 and certs[1]["cycle"] >= 2     # the 2-cycle's edges attain the distances


def _errors_worker(rank, world, s, d, w):
    import torch
    from cugraph_b200 import mg
    g = mg_world.graph(rank, world, s, d, w)
    v, dd, pp = g.bfs(int(s[0]))
    out = []
    for args in ((v, dd, None), (v, dd[:-1] if rank == 0 else dd, pp), (v.long(), dd, pp), (v, dd.float(), pp)):
        try:
            g.validate_bfs(*args, int(s[0]))
            out.append(None)
        except (TypeError, ValueError) as e:
            out.append(type(e).__name__)
    gu = mg_world.graph(rank, world, s, d)
    try:
        gu.validate_sssp(v, dd.float(), pp, int(s[0]))
    except ValueError as e:
        out.append(str(e))
    del torch
    return out


def test_certificate_errors_on_every_rank(surface, monkeypatch):  # noqa: F811
    s, d, w, V = mg_sssp_ref.rmat_graph(8, np.float32)
    res = mg_world.run(mg_world.grid_world(monkeypatch, 2, 2), _errors_worker, s, d, w)
    for r in res:
        assert r == ["ValueError", "ValueError", "TypeError", "TypeError", "SSSP requires a weighted graph"]


# ---------------------------------------------------------------------------------------------------------- harness
def _harness_worker(rank, world):
    from cugraph_b200 import mg
    from scripts.graph500 import run
    return run(mg.make_groups(), 8, n_roots=4)


def test_harness_emulated_gloo():
    res = mg_procs.run(_harness_worker, 2, emulated=True, timeout=600)
    out = res[0]
    timing = {"construction_s", "time_s", "teps", "validation_s_per_root"}   # maxed over ranks, the rest is exact

    def exact(d):
        return {k: exact(v) if isinstance(v, dict) else v for k, v in d.items() if k not in timing}
    assert exact(res[0]) == exact(res[1])
    assert all(r[k][t] == out[k][t] for r in res for k in ("bfs", "sssp") for t in ("time_s", "teps"))
    assert out["ok"] and out["grid"] == "2x1" and out["roots"] == 4 and out["scale"] == 8 and out["edge_factor"] == 16
    for k in ("bfs", "sssp"):
        assert out[k]["validated"] == out[k]["roots"] == 4
        assert set(out[k]["time_s"]) == {"min", "q1", "median", "q3", "max", "mean", "stddev"}
        assert set(out[k]["teps"]) >= {"harmonic_mean", "harmonic_stddev"}
        assert out[k]["validation_s_per_root"] >= 0
    assert out["construction_s"] > 0
