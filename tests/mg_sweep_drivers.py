"""The multi-GPU drivers of the block sweep — MGGraph.pagerank (plain, personalized, from an initial guess, with precomputed
out-weights), .katz_centrality, .eigenvector_centrality and .hits — checked step for step against the fp64 references of
tests/sweep_drivers.py: the harness of tests/test_mg_sweep_drivers_gpu.py (the H100) and tests/test_mg_sweep_drivers_cpu.py
(the emulation build of the library).

The graph of a case is directed RMAT with multi-edges and self-loops kept; its vertices are the ids that appear in edges,
which is what an MGGraph has, so the reference sweep_drivers.Graph is built over those ids (internal id = rank among them,
external id = the RMAT id, or a scattered int64 id).  Every rank of the grid builds its MGGraph from its share of the edge
list under the case's CUGRAPH_B200_* knobs (read once, when the graph's handle is created) and runs the same calls on it in
order; the results are gathered by vertex and handed to sweep_drivers.verify_*, with the iteration counts the drivers
report and the extra rounding of the reduce-scatter: (G - 1) u per sweep, G the size of the group that reduce-scatters it
(the row group, C, for the pull sweep; the column group, R, for HITS' transposed sweep) — see sweep_drivers' docstring.

Grids: R x C simulated in ONE process (tests/mg_world.py: one thread per rank, the collectives an in-process stand-in), or
one process per GPU over NCCL (tests/mg_procs.py; gloo over the emulated library on the CPU).  Layouts: every rank's block must have built the piece streams its
knobs ask for — sweep_rows.expected_layout of the block's row counts (cugraph_b200_block_degrees), and once HITS has run,
of its column counts for the transposed copy — and a layout that asks for a piece stream must get one on every block
with edges, so that a case cannot pass on the plain sweep.  CUGRAPH_B200_BUILD_TRACE=1 prints what was built: on the
simulated grid all ranks write to one stderr (the traces are matched as a multiset), in a process group each rank captures
its own."""
import contextlib
import os

import numpy as np

from tests import mg_world
from tests import sweep_drivers as sd
from tests import sweep_rows as sr

GRIDS = {"1x2": (1, 2), "2x1": (2, 1), "2x2": (2, 2), "4x2": (4, 2)}
KNOBS = dict(sd.KNOBS, default={})     # default: no knobs, the layout the library picks by itself
PREFIX = "mg "                  # the keys of sweep_drivers.WORST that the multi-GPU checks record


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
_GRAPHS = {}


def over_present(s, d, T, w, scattered_ids=False, seed=0, label=""):
    """the Graph over the ids that appear in the edge list s -> d (internal id = rank among them); external ids are those
    ids (int32), or scattered int64 ids"""
    ids, remap = mg_world.present(s, d, int(max(s.max(), d.max())) + 1)
    ext = ids.astype(np.int32)
    if scattered_ids:
        ext = np.random.default_rng(seed + 1).choice(np.arange(10**12, 10**12 + 10**8), ids.size,
                                                     replace=False).astype(np.int64)
    return sd.Graph(remap[s], remap[d], ids.size, T, w, "csc", ext, label)


def graph_of(etype, scale, scattered_ids=False):
    """directed RMAT at `scale` (the emulation's cap applied) over its present ids, cached per module run"""
    from oracle.rmat import rmat_edgelist
    scale = sd.scale_of(scale)
    key = (etype, scale, scattered_ids)
    if key not in _GRAPHS:
        T, weighted = sd.TYPES[etype]
        seed = 1900 + scale + (17 if scattered_ids else 0)
        s, d = rmat_edgelist(scale, 16 << scale, seed=seed)
        s, d = np.asarray(s, np.int64), np.asarray(d, np.int64)
        w = np.random.default_rng(seed).uniform(0.5, 1.0, s.size).astype(T) if weighted else None
        _GRAPHS[key] = over_present(s, d, T, w, scattered_ids=scattered_ids, seed=seed,
                                    label=f"RMAT-{scale} {np.dtype(T).name}{'w' if weighted else ''}"
                                          f"{' int64-ids' if scattered_ids else ''}")
    return _GRAPHS[key]


# ---------------------------------------------------------------------------------------------------------------------
# the calls: dicts with "algo" and its arguments, pairs (ids, values) in internal ids
# ---------------------------------------------------------------------------------------------------------------------
def pagerank_calls(graph, steps):
    """plain, each personalization, and an initial guess with precomputed out-weights (twice the true sums) and the
    personalization with zeros among its values"""
    pers = sd.personalizations(graph)
    calls = [dict(algo="pagerank", steps=steps)]
    calls += [dict(algo="pagerank", steps=steps, pers=p, name=n) for n, p in pers.items()]
    rng = np.random.default_rng(4)
    guess = (np.arange(graph.V), rng.uniform(0.0, 2.0 / graph.V, graph.V).astype(graph.T))
    calls.append(dict(algo="pagerank", steps=steps, pers=pers["share_with_zeros"], guess=guess,
                      out_w=out_weights(graph, 2.0)))
    return calls


def out_weights(graph, factor=1.0):
    ow = np.bincount(graph.s, weights=None if graph.w is None else graph.w.astype(np.float64), minlength=graph.V)
    return np.arange(graph.V), (factor * ow).astype(graph.T)


def katz_calls(graph):
    eps = sd.epsilons(graph)["katz"]
    return [dict(algo="katz", alpha=sd.katz_alpha(graph), epsilon=eps),
            dict(algo="katz", alpha=sd.katz_alpha(graph, 0.9), epsilon=eps, near=True)]


def hits_calls(graph):
    eps = sd.epsilons(graph)["hits"]
    rng = np.random.default_rng(3)
    part = np.sort(rng.choice(graph.V, graph.V // 3, replace=False))
    guess = (part, rng.uniform(0.1, 1.0, part.size).astype(graph.T))
    return [dict(algo="hits", epsilon=eps, guess=g, normalize=n) for g in (None, guess) for n in (True, False)]


def all_calls(graph, steps):
    eps = sd.epsilons(graph)
    return (pagerank_calls(graph, steps) + katz_calls(graph) + [dict(algo="eigenvector", epsilon=eps["eigenvector"])]
            + hits_calls(graph))


def many_calls(graph, steps=30):
    """single GPU's run_many_calls on one MGGraph: PageRank, Katz, HITS, eigenvector, personalized PageRank, PageRank with
    precomputed out-weights (twice the true sums), plain PageRank again"""
    eps = sd.epsilons(graph)
    return [dict(algo="pagerank", steps=steps), katz_calls(graph)[0], dict(algo="hits", epsilon=eps["hits"]),
            dict(algo="eigenvector", epsilon=eps["eigenvector"]),
            dict(algo="pagerank", steps=steps, pers=sd.personalizations(graph)["share_with_zeros"]),
            dict(algo="pagerank", steps=steps, out_w=out_weights(graph, 2.0)), dict(algo="pagerank", steps=steps)]


def _external(graph, call):
    """the call with its (internal ids, values) pairs in external ids"""
    return {k: (graph.ext(np.asarray(v[0])), v[1]) if k in ("pers", "guess", "out_w") and v is not None else v
            for k, v in call.items()}


# ---------------------------------------------------------------------------------------------------------------------
# one rank
# ---------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _stderr_text(on):
    """with `on`, fd 2 goes to a temporary file inside the block; the list it yields then receives the text"""
    import sys
    import tempfile
    out = []
    if not on:
        yield out
        return
    sys.stderr.flush()
    saved = os.dup(2)
    with tempfile.TemporaryFile() as f:
        os.dup2(f.fileno(), 2)
        try:
            yield out
        finally:
            os.dup2(saved, 2)
            os.close(saved)
            f.seek(0)
            out.append(f.read().decode(errors="replace"))


def _block_degrees(g):
    """the entries of every row and every column slot of this rank's block"""
    import torch
    from cugraph_b200 import mg
    rows = torch.empty(g.n_rows, dtype=torch.int64, device=g.device)
    cols = torch.empty(g.n_cols, dtype=torch.int64, device=g.device)
    with mg._views(rows, cols) as (vr, vc):
        g._call("cugraph_b200_block_degrees", g.block, vr.ptr, vc.ptr)
    return rows.cpu().numpy(), cols.cpu().numpy()


def _np(t):
    return t.cpu().numpy()


def _one_call(g, rank, world, c):
    share = (lambda p: None if p is None else mg_world.share(rank, world, *p))   # pairs spread over the ranks
    algo = c["algo"]
    if algo == "pagerank":
        v, x, it, _ = g.pagerank(alpha=c.get("alpha", 0.85), epsilon=0.0, max_iterations=c["steps"],
                                 personalization=share(c.get("pers")), initial_guess=share(c.get("guess")),
                                 precomputed_out_weights=share(c.get("out_w")))
        return _np(v), (_np(x),), dict(iterations=it)
    if algo == "katz":
        v, x = g.katz_centrality(c["alpha"], beta=1.0, epsilon=c["epsilon"], max_iterations=1000)
        return _np(v), (_np(x),), dict(g.last_katz_stats)
    if algo == "eigenvector":
        v, x = g.eigenvector_centrality(epsilon=c["epsilon"], max_iterations=1000)
        return _np(v), (_np(x),), dict(g.last_eigenvector_stats)
    v, hb, au = g.hits(epsilon=c["epsilon"], max_iterations=1000, initial_hubs_guess=share(c.get("guess")),
                       normalize=c.get("normalize", True))
    return _np(v), (_np(hb), _np(au)), dict(g.last_hits_stats)


def worker(rank, world, s, d, w, T, calls, capture=False):
    """rank's MGGraph from its share of the edges (external ids), the calls on it in order; returns the results, the
    block's row / column counts and edges, and with `capture` the rank's own stderr"""
    device = "cpu" if sd.emulated() else "cuda"
    with _stderr_text(capture) as text:
        g = mg_world.graph(rank, world, s, d, w, T, device)
        rows, cols = _block_degrees(g)
        out = [_one_call(g, rank, world, c) for c in calls]
        res = dict(out=out, rows=rows, cols=cols, nnz=g.num_edges_local, span=g.span)
        del g
    res["trace"] = text[0] if text else None
    return res


# ---------------------------------------------------------------------------------------------------------------------
# a grid
# ---------------------------------------------------------------------------------------------------------------------
def set_knobs(monkeypatch, knobs):
    for k in sr.KNOBS:
        monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)
    for k, v in knobs.items():
        monkeypatch.setenv("CUGRAPH_B200_" + k, str(v))
    monkeypatch.setenv("CUGRAPH_B200_BUILD_TRACE", "1")


def run(monkeypatch, capfd, graph, layout, grid, calls):
    """the calls on one MGGraph per rank of `grid` ("RxC": simulated in this process; "nccl-N": N processes, one GPU each;
    "gloo-N": N processes over the emulated library)
    built under KNOBS[layout], each result verified, the blocks' layouts checked; returns (the worst observed / bound,
    [(edges, [layouts built]) of every rank's block])"""
    from cugraph_b200 import mg
    from tests import mg_procs
    knobs = KNOBS[layout]
    s, d = graph.ext(graph.s), graph.ext(graph.d)
    ext_calls = [_external(graph, c) for c in calls]
    set_knobs(monkeypatch, knobs)
    capfd.readouterr()
    try:
        if grid.startswith(("nccl-", "gloo-")):
            backend, world = grid[:4], int(grid[5:])
            monkeypatch.delenv("CUGRAPH_B200_MG_GRID", raising=False)
            R, Cc = mg.grid_shape(world)
            env = {"CUGRAPH_B200_" + k: str(v) for k, v in knobs.items()}
            res = mg_procs.run(worker, world, s, d, graph.w, graph.T, ext_calls, True, backend=backend,
                               emulated=backend == "gloo", env=env, timeout=900)
        else:
            R, Cc = GRIDS[grid]
            world = mg_world.grid_world(monkeypatch, R, Cc)
            res = mg_world.run(world, worker, s, d, graph.w, graph.T, ext_calls)
    finally:
        for k in list(knobs) + ["BUILD_TRACE"]:
            monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)
    label = f"{grid} {layout}"
    wants = check_layouts(res, capfd.readouterr().err, graph, layout, any(c["algo"] == "hits" for c in calls), label)
    u = sd.unit(graph.T)
    extra_pull, extra_tr = (Cc - 1) * u, (R - 1) * u
    worst = 0.0
    for k, c in enumerate(calls):
        worst = max(worst, verify(graph, c, [r["out"][k] for r in res], extra_pull, extra_tr, grid, label))
    return worst, [(r["nnz"], w) for r, w in zip(res, wants)]


def verify(graph, c, parts, extra_pull, extra_tr, grid, label):
    """one call's results from every rank against its reference"""
    import torch
    verts = np.concatenate([p[0] for p in parts])
    stats = parts[0][2]
    assert all(p[2] == stats for p in parts), f"{label}: the ranks report different {[p[2] for p in parts]}"
    vals = [graph.dense(torch.from_numpy(verts), torch.from_numpy(np.concatenate([p[1][j] for p in parts])))
            for j in range(len(parts[0][1]))]
    t = np.dtype(graph.T).name
    tag = f" on {label}"
    k = stats["iterations"]
    algo = c["algo"]
    if algo == "pagerank":
        key = f"{PREFIX}{'personalized ' if c.get('pers') is not None else ''}pagerank {t} {grid}"
        name = f" ({c['name']})" if "name" in c else ""
        return sd.verify_pagerank(graph, vals[0], k, c["steps"], c.get("alpha", 0.85), c.get("pers"), c.get("guess"),
                                  c.get("out_w"), extra=extra_pull, key=key, tag=tag + name)
    if algo == "katz":
        key = f"{PREFIX}katz {t}{' near the limit' if c.get('near') else ''} {grid}"
        return sd.verify_katz(graph, vals[0], k, c["alpha"], 1.0, c["epsilon"], extra=extra_pull, key=key, tag=tag)
    if algo == "eigenvector":
        key = f"{PREFIX}eigenvector {t} {grid}"
        return sd.verify_eigenvector(graph, vals[0], k, c["epsilon"], extra=extra_pull, key=key, tag=tag)
    return sd.verify_hits(graph, vals[0], vals[1], stats["hub_score_differences"], k, c["epsilon"], c.get("guess"),
                          c.get("normalize", True), extra=(extra_pull, extra_tr), key=f"{PREFIX}hits {t} {grid}", tag=tag)


# ---------------------------------------------------------------------------------------------------------------------
# layouts
# ---------------------------------------------------------------------------------------------------------------------
def block_layouts(r, knobs, es, transposed):
    """the piece streams rank result `r`'s block must have built: its pull layout and, once HITS has swept it,
    the layout of its column-major copy (None: the plain sweep)"""
    span = r["span"]
    pad = (lambda c: np.concatenate([c, np.zeros(span - c.size, np.int64)]))
    views = [r["rows"]] + ([r["cols"]] if transposed else [])
    return [sr.expected_layout(pad(c), r["nnz"], knobs, es, sd.l2_bytes()) for c in views]


def _trace_key(seg):
    m, t = sr._HEAD.search(seg), sr._TAIL.search(seg)
    return tuple(map(int, m.groups())) + (tuple(map(int, t.groups())) if t else (),)


def _want_key(w):
    tail = (w["runs"], w["tiles"], w["units"]) if w["tail"] else ()
    return (w["B"], w["W"], w["rows"], w["tail"], w["bands"], w["band_rows"], tail)


def match_traces(err, wants, label):
    """the piece streams traced in `err` are exactly those of `wants`, in any order"""
    starts = [m.start() for m in sd._HEAD.finditer(err)]
    got = sorted(_trace_key(err[a:b]) for a, b in zip(starts, starts[1:] + [len(err)]))
    want = sorted(_want_key(w) for w in wants if w is not None)
    assert got == want, (f"{label}: piece streams built (B, W, rows, tail, bands, band rows, (tail runs, tiles, units)):\n"
                         f"  {got}\nexpected:\n  {want}\n{err}")


def check_layouts(res, err, graph, layout, transposed, label):
    """every block built the layouts its knobs ask for; a layout that asks for a piece stream got one on every block
    with edges (in both orientations, once HITS ran), and bands-tail a tail on some block"""
    knobs = KNOBS[layout]
    es = np.dtype(graph.T).itemsize
    wants = [block_layouts(r, knobs, es, transposed) for r in res]
    if res[0]["trace"] is not None:
        for rank, (r, w) in enumerate(zip(res, wants)):
            match_traces(r["trace"], w, f"{label} rank {rank}")
    else:
        match_traces(err, [x for w in wants for x in w], label)
    flat = [x for r, w in zip(res, wants) for x in w if r["nnz"] > 0]
    if layout in ("stream", "bands-tail", "default"):
        assert flat and all(x is not None for x in flat), f"{label}: a block with edges runs the plain sweep: {wants}"
    if layout == "bands-tail":
        assert any(x["tail"] > 0 for x in flat), f"{label}: no block has a tail: {wants}"
    if layout in ("plain", "offs64"):
        assert all(x is None for x in flat), f"{label}: {wants}"
    return wants


def report(request, title):
    """print the multi-GPU margins on record past pytest's output capture, and drop them from sweep_drivers.WORST"""
    capman = request.config.pluginmanager.getplugin("capturemanager")
    keys = sorted(k for k in sd.WORST if k.startswith(PREFIX))
    if keys and capman is not None:
        with capman.global_and_fixture_disabled():
            print(f"\n{title}")
            for k in keys:
                print(f"  {k[len(PREFIX):]:<48} {sd.WORST[k]:.3e}")
    for k in keys:
        del sd.WORST[k]
