"""Multi-GPU PageRank with personalization, an initial guess and precomputed out-weights on the CPU, over the emulated
library (tests/emu_py.py).

- Every rank of a grid in one process (tests/mg_world.py) running cugraph_b200.mg.MGGraph.pagerank: grids 1x2, 2x1, 2x2
  and 4x2 on a directed RMAT-8 and on a graph with isolated ids, sources, sinks and duplicate edges, weighted and
  unweighted, float32 and float64, against the fp64 oracle on the graph's vertices at equal iteration count.
- The personalized owner step's entry point: its arithmetic and its error paths.
- World sizes 2, 4 and 8 over gloo running MGGraph.pagerank (the real process groups): personalization from one rank,
  from a rank that owns none of its vertices and split across ranks; the reference's two personalized C-API goldens with
  the personalization given by rank 0 only; an initial guess and precomputed out-weights; every input error raised on
  every rank with the same type and message; FailedToConvergeError on every rank."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import mg_centrality_ref as graphs  # noqa: E402
from tests import mg_pagerank_ref as refs  # noqa: E402
from tests import mg_procs  # noqa: E402
from tests import mg_world  # noqa: E402
from tests.emu_py import surface  # noqa: E402, F401

GRIDS = [(1, 2), (2, 1), (2, 2), (4, 2)]
GRID_IDS = ["1x2", "2x1", "2x2", "4x2"]
ITERS = 20


def check_all(s, d, V, world, w=None, dtype=np.float32, device="cpu", iters=ITERS, single=False):
    """plain and personalized runs, doubled out-weights and a converged initial guess on one grid against the oracle (and,
    with `single`, against single-GPU personalized PageRank), all on the vertices that appear in edges"""
    tol = refs.F64_TOL if dtype == np.float64 else refs.F32_TOL
    ids, remap = mg_world.present(s, d, V)
    rs, rd, n = remap[s], remap[d], ids.size
    ow = refs.out_weights(rs, n, w)
    # dense over the vertices; the isolated id's case personalizes no vertex of the graph
    pers = {name: pv[ids] for name, pv in refs.cases(s, d, V).items() if pv[ids].any()}
    share = pers["share_with_zeros"]
    conv_ref = {k: refs.oracle_pagerank(rs, rd, n, w, epsilon=1e-12, max_iterations=1000, personalization=pv)[0]
                for k, pv in (("plain", None), ("share", share))}
    fixed = dict(alpha=0.85, epsilon=0.0, max_iterations=iters)
    runs = [fixed] + [dict(fixed, personalization=(ids, pv)) for pv in pers.values()]
    runs += [dict(fixed, personalization=(ids, np.ones(n))), dict(fixed, precomputed_out_weights=(ids, 2.0 * ow))]
    runs += [dict(alpha=0.85, epsilon=1e-5, max_iterations=100, initial_guess=(ids, conv_ref["plain"])),
             dict(alpha=0.85, epsilon=1e-5, max_iterations=100, initial_guess=(ids, conv_ref["share"]),
                  personalization=(ids, share))]
    got = [(x[ids], it, conv) for x, it, conv in refs.mg_pagerank(s, d, V, world, runs, w=w, dtype=dtype, device=device)]
    plain, it, conv = got[0]
    assert it == iters and not conv
    np.testing.assert_allclose(plain, refs.oracle_pagerank(rs, rd, n, w, max_iterations=iters)[0], **tol)
    for (name, pv), (x, _, _) in zip(pers.items(), got[1:]):
        want, _, _ = refs.oracle_pagerank(rs, rd, n, w, max_iterations=iters, personalization=pv)
        np.testing.assert_allclose(x, want, **tol, err_msg=name)
        if single:
            np.testing.assert_allclose(x, single_gpu(rs, rd, n, w, pv, iters), **tol, err_msg=name)
    ones, doubled, from_plain, from_share = got[len(pers) + 1:]
    np.testing.assert_allclose(ones[0], plain, **tol)               # teleport to every vertex alike = plain PageRank
    want, _, _ = refs.oracle_pagerank(rs, rd, n, w, max_iterations=iters, out_w=2.0 * ow)
    np.testing.assert_allclose(doubled[0], want, **tol)
    for (x, it, conv), k in ((from_plain, "plain"), (from_share, "share")):
        assert it == 1 and conv
        np.testing.assert_allclose(x, conv_ref[k], rtol=1e-5, atol=1e-12)


def single_gpu(s, d, V, w, pv, iters):
    """single-GPU cugraph_personalized_pagerank_allow_nonconvergence with the same personalization, by vertex id"""
    import torch
    from cugraph_b200 import pylibcugraph as plc
    from tests.gpu_util import by_vertex, make_graph
    wdt = np.float32 if w is None else w.dtype
    h, g = make_graph(s, d, weights=w, store_transposed=True, vertices=np.arange(V, dtype=np.int32), weight_dtype=wdt)
    ids = np.flatnonzero(pv != 0).astype(np.int32)
    v, x, _ = plc.personalized_pagerank(h, g, None, None, None, None, torch.as_tensor(ids).cuda(),
                                        torch.as_tensor(pv[ids].astype(wdt)).cuda(), 0.85, 0.0, iters, False,
                                        fail_on_nonconvergence=False)
    return by_vertex(v, x, V).astype(np.float64)


@pytest.mark.parametrize("R,Cc", GRIDS, ids=GRID_IDS)
def test_mg_pagerank_simulated_emulated(surface, monkeypatch, R, Cc):
    world = mg_world.grid_world(monkeypatch, R, Cc)
    check_all(*graphs.rmat_graph(8), world)
    check_all(*graphs.odd_graph(), world)


@pytest.mark.parametrize("wdtype", [np.float32, np.float64], ids=["f32", "f64"])
def test_mg_pagerank_weighted_emulated(surface, monkeypatch, wdtype):
    s, d, V = graphs.odd_graph()
    w = np.random.default_rng(2).uniform(0.5, 1.0, s.size).astype(wdtype)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 2, 2), w=w, dtype=wdtype)


def test_mg_pagerank_float64_rmat_emulated(surface, monkeypatch):
    s, d, V = graphs.rmat_graph(8)
    w = np.random.default_rng(3).uniform(0.5, 1.0, s.size)
    check_all(s, d, V, mg_world.grid_world(monkeypatch, 4, 2), w=w, dtype=np.float64)


def test_personalized_vertex_step_emulated(surface):
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    handle = ResourceHandle(stream=0)
    tot = torch.tensor([0.0, 0.25], dtype=torch.float64)           # previous step: dangling sum 0.25
    part = torch.zeros(2, dtype=torch.float64)
    tp, pp = C.c_void_p(tot.data_ptr()), C.c_void_p(part.data_ptr())

    def call(*args):
        views = [View(a) if isinstance(a, torch.Tensor) else a for a in args]
        err = C.c_void_p()
        code = L.cugraph_b200_pagerank_personalized_vertex_step(
            handle.ptr, *[v.ptr if isinstance(v, View) else v for v in views], C.byref(err))
        for v in views:
            if isinstance(v, View):
                v.free()
        _capi.check(code, err, "cugraph_b200_pagerank_personalized_vertex_step")

    y = torch.tensor([0.1, 0.2, 0.3, 0.4], dtype=torch.float64)
    pr = torch.tensor([0.25, 0.25, 0.25, 0.25], dtype=torch.float64)
    ow = torch.tensor([1.0, 2.0, 0.0, 4.0], dtype=torch.float64)
    x = torch.zeros(4, dtype=torch.float64)
    pers = torch.tensor([1.0, 0.0, 3.0, 0.0], dtype=torch.float64)
    alpha = 0.85
    call(y, pr, ow, x, pers, 4, alpha, 4.0, 0, tp, pp)
    base = 0.25 * alpha + (1.0 - alpha)
    want = y.numpy() + base * (pers.numpy() / 4.0)
    np.testing.assert_array_equal(pr.numpy(), want)
    np.testing.assert_array_equal(x.numpy(), np.where(ow.numpy() == 0, want, want / np.where(ow.numpy() == 0, 1, ow.numpy())))
    assert part[0].item() == pytest.approx(np.abs(want - 0.25).sum()) and part[1].item() == want[2]
    # first = TRUE: pr unchanged, no totals read
    part.zero_()
    pr2 = pr.clone()
    call(y, pr2, ow, x, pers, 4, alpha, 4.0, 1, None, pp)
    assert torch.equal(pr2, pr) and part[0].item() == 0.0
    # the errors: NULL pers / totals, dtype, short arrays, pers_sum <= 0, NaN pers_sum
    for args in ((y, pr, ow, x, None, 4, alpha, 4.0, 0, tp, pp), (y, pr, ow, x, pers, 4, alpha, 4.0, 0, None, pp),
                 (y, pr, ow, x, pers.float(), 4, alpha, 4.0, 0, tp, pp), (y, pr, ow, x, pers[:3], 4, alpha, 4.0, 0, tp, pp),
                 (y, pr, ow, x, pers, 4, alpha, 0.0, 0, tp, pp), (y, pr, ow, x, pers, 4, alpha, -1.0, 0, tp, pp),
                 (y, pr, ow, x, pers, 4, alpha, float("nan"), 0, tp, pp), (y, pr, ow, x, pers, 4, alpha, 4.0, 0, tp, None)):
        with pytest.raises(_capi.CugraphError) as e:
            call(*args)
        assert e.value.code == _capi.INVALID_INPUT
    call(y[:0], pr[:0], ow[:0], x[:0], pers[:0], 0, alpha, 4.0, 0, tp, pp)    # an owner without vertices


# ---------------------------------------------------------------------------------------------------------- gloo runs
def _gloo_graph():
    """the odd graph with scattered 64-bit external ids (isolated ids are not vertices of an MG graph)"""
    s, d, V = graphs.odd_graph(seed=13)
    ids = np.random.default_rng(13).choice(10**9, size=V, replace=False).astype(np.int64) + 10**10
    return ids, s, d, V


def _inputs(ids, s, d):
    """personalization on a random share of the vertices, one vertex, an initial guess and out-weights, by external id"""
    rng = np.random.default_rng(21)
    present = np.unique(np.concatenate([s, d]))
    share = rng.choice(present, size=present.size // 4, replace=False)
    guess = rng.uniform(0.0, 2.0 / present.size, present.size)
    ow = np.bincount(s, minlength=ids.size).astype(np.float64)[present] * 1.5
    return dict(share=(ids[share], rng.uniform(0.0, 1.0, share.size)), one=(ids[present[:1]], np.array([2.0])),
                guess=(ids[present], guess), ow=(ids[present], ow), present=present)


def _split(pair, rank, world):
    """rank's slice of a pair: the pairs spread over all ranks"""
    n = pair[0].size
    lo, hi = rank * n // world, (rank + 1) * n // world
    return pair[0][lo:hi], pair[1][lo:hi]


def _error_cases(ids, rank, world):
    """(name, kwargs of MGGraph.pagerank on this rank) for every row of the input-error table"""
    last = world - 1
    a, b = int(ids[0]), int(ids[1])
    e = np.zeros(0, np.int64), np.zeros(0)
    only = (lambda r, pair: pair if rank == r else None)
    # the same id from the first and the last rank (twice from the one rank of a world of one)
    dup = (np.array([a] * (2 if world == 1 else 1)), np.array([1.0] * (2 if world == 1 else 1))) if rank in (0, last) else None
    return [
        ("pers_size", dict(personalization=only(min(1, last), (np.array([a, b]), np.array([1.0]))))),
        ("pers_empty", dict(personalization=only(0, e))),
        ("pers_invalid", dict(personalization=only(0, (np.array([a, 5]), np.array([1.0, 1.0]))))),
        ("pers_negative", dict(personalization=only(last, (np.array([a, b]), np.array([1.0, -1.0]))))),
        ("pers_duplicate", dict(personalization=dup)),
        ("pers_zero_sum", dict(personalization=only(0, (np.array([a, b]), np.array([0.0, 0.0]))))),
        ("guess_size", dict(initial_guess=only(last, (np.array([a, b]), np.array([1.0]))))),
        ("guess_invalid", dict(initial_guess=only(0, (np.array([a, 7]), np.array([1.0, 1.0]))))),
        ("ow_size", dict(precomputed_out_weights=only(0, (np.array([a]), np.array([1.0, 2.0]))))),
        ("ow_invalid", dict(precomputed_out_weights=only(last, (np.array([9]), np.array([1.0]))))),
    ]


def _golden_worker_part(rank, golden, device):
    """the reference's MG C test: personalization from rank 0 only"""
    import torch
    from cugraph_b200 import mg
    out = {}
    for case in ("personalized_pagerank_4", "personalized_pagerank_4_nonconverged"):
        c = golden[case]
        src, dst = np.asarray(c["src"], np.int64), np.asarray(c["dst"], np.int64)
        n = src.size
        world = torch.distributed.get_world_size()
        lo, hi = rank * n // world, (rank + 1) * n // world
        g = mg.MGGraph(torch.from_numpy(src[lo:hi]).to(device), torch.from_numpy(dst[lo:hi]).to(device),
                       torch.tensor(c["weights"][lo:hi], dtype=torch.float32).to(device))
        pers = (np.asarray(c["personalization_vertices"]), np.asarray(c["personalization_values"])) if rank == 0 else None
        v, x, conv = mg.personalized_pagerank(g, pers, c["alpha"], c["epsilon"], c["max_iterations"])
        out[case] = (v.cpu().numpy(), x.cpu().numpy(), conv)
    return out


def _gloo_worker(rank, world, golden, device="cpu"):
    """the MGGraph runs of one rank (device "cuda" under NCCL)"""
    import torch
    from cugraph_b200 import mg
    from cugraph_b200.pylibcugraph.exceptions import FailedToConvergeError
    ids, s, d, V = _gloo_graph()
    n = s.size
    lo, hi = rank * n // world, (rank + 1) * n // world
    g = mg.MGGraph(torch.from_numpy(ids[s[lo:hi]]).to(device), torch.from_numpy(ids[d[lo:hi]]).to(device))
    inp = _inputs(ids, s, d)
    out = {}

    def run(key, **kw):
        v, x, it, conv = g.pagerank(0.85, 0.0, ITERS, **kw)
        out[key] = (v.cpu().numpy(), x.cpu().numpy(), it, conv)

    run("plain")
    run("share_rank0", personalization=inp["share"] if rank == 0 else None)
    run("share_split", personalization=_split(inp["share"], rank, world))
    one_owner = int(mg.vertex_owner(torch.from_numpy(inp["one"][0]), world)[0])
    run("one_not_owner", personalization=inp["one"] if rank == (one_owner + 1) % world else None)
    run("guess_ow", initial_guess=_split(inp["guess"], rank, world),
        precomputed_out_weights=inp["ow"] if rank == world - 1 else None)
    true_ow = (inp["ow"][0], inp["ow"][1] / 1.5)
    run("true_ow", precomputed_out_weights=_split(true_ow, rank, world))
    out["golden"] = _golden_worker_part(rank, golden, device)
    errs = {}
    for name, kw in _error_cases(ids, rank, world):
        try:
            g.pagerank(0.85, 0.0, 3, **kw)
            errs[name] = None
        except Exception as e:  # noqa: BLE001
            errs[name] = (type(e).__name__, str(e))
    try:
        g.pagerank(0.85, 1e-12, 2, personalization=inp["share"] if rank == 0 else None, fail_on_nonconvergence=True)
        errs["nonconvergence"] = None
    except FailedToConvergeError as e:
        errs["nonconvergence"] = (type(e).__name__, str(e))
    out["errors"] = errs
    return out


ERROR_TABLE = {
    "pers_size": ("CugraphRuntimeError", "the size of vertices and values should match"),
    "pers_empty": ("CugraphRuntimeError", "the input personalization vector size should not be 0."),
    "pers_invalid": ("CugraphValueError", "peresonalization vertices have invalid vertex IDs."),
    "pers_negative": ("CugraphValueError", "peresonalization values should be non-negative."),
    "pers_duplicate": ("CugraphValueError", "personalization vertices should not contain duplicate entries."),
    "pers_zero_sum": ("CugraphRuntimeError", "sum of personalization valuese should be positive."),
    "guess_size": ("CugraphValueError", "initial_guess: vertex and value arrays differ in size"),
    "guess_invalid": ("CugraphValueError", "initial_guess: vertex list contains ids that are not vertices of the graph"),
    "ow_size": ("CugraphValueError", "precomputed_out_weights: vertex and value arrays differ in size"),
    "ow_invalid": ("CugraphValueError",
                   "precomputed_out_weights: vertex list contains ids that are not vertices of the graph"),
    "nonconvergence": ("FailedToConvergeError", "PageRank failed to converge"),
}


def check_gloo(res, ids, s, d, V, golden, tol):
    """every rank's results of _gloo_worker against the oracle on the graph's vertex set, and the error table"""
    inp = _inputs(ids, s, d)
    present = inp["present"]
    k_of = {int(ids[v]): i for i, v in enumerate(present)}
    remap = np.full(V, -1)
    remap[present] = np.arange(present.size)
    rs, rd, n = remap[s], remap[d], present.size

    def dense(pair):
        out = np.zeros(n)
        out[[k_of[int(x)] for x in pair[0]]] = pair[1]
        return out

    def by_id(key):
        out = np.zeros(n)
        cnt = 0
        for r in res:
            v, x = r[key][0], r[key][1]
            out[[k_of[int(e)] for e in v]] = x
            cnt += v.size
        assert cnt == n
        assert all(r[key][2] == ITERS and not r[key][3] for r in res)
        return out

    def ref(**kw):
        return refs.oracle_pagerank(rs, rd, n, max_iterations=ITERS, **kw)[0]

    np.testing.assert_allclose(by_id("plain"), ref(), **tol)
    np.testing.assert_allclose(by_id("share_rank0"), ref(personalization=dense(inp["share"])), **tol)
    np.testing.assert_allclose(by_id("share_split"), ref(personalization=dense(inp["share"])), **tol)
    np.testing.assert_allclose(by_id("one_not_owner"), ref(personalization=dense(inp["one"])), **tol)
    np.testing.assert_allclose(by_id("guess_ow"), ref(initial_guess=dense(inp["guess"]), out_w=dense(inp["ow"])), **tol)
    assert np.array_equal(by_id("true_ow"), by_id("plain"))       # the true sums: bit-identical to the derived ones
    for case in ("personalized_pagerank_4", "personalized_pagerank_4_nonconverged"):
        c = golden[case]
        got = np.zeros(c["num_vertices"])
        for r in res:
            v, x, conv = r["golden"][case]
            got[v] = x
            assert conv == ("nonconverged" not in case)
        np.testing.assert_allclose(got, c["values"], rtol=c["rel_tol"])
    for name, (cls, msg) in ERROR_TABLE.items():
        first = res[0]["errors"][name]
        assert first is not None and first[0] == cls and msg in first[1], (name, first)
        assert all(r["errors"][name] == first for r in res), name      # the same exception on every rank


@pytest.mark.parametrize("world", [2, 4, 8])
def test_mg_pagerank_emulated_gloo(world, golden):
    res = mg_procs.run(_gloo_worker, world, golden["c_api"], emulated=True)
    ids, s, d, V = _gloo_graph()
    check_gloo(res, ids, s, d, V, golden["c_api"], dict(rtol=1e-5, atol=1e-12))
