"""PageRank with its vertex pass done by the pull sweep's row epilogue (sweep_epilogue_t: next x, dangling sum and, at
epsilon > 0, the difference, computed where each row is written) on the H100, on every sweep layout: the plain sweep with
32- and 64-bit offsets, the piece stream, the piece stream in forced bands with a tail, and the re-sorted (row_vertex) pull
view of a CSR graph.  Each check runs PageRank for a number of steps and compares with an fp64 reference after exactly that
many (odd and even counts: the two x buffers alternate), at epsilon = 0 and at epsilon > 0, where the iteration count and
the converged flag must be the reference's.  float32 and float64, weighted and unweighted, with an initial guess,
precomputed out-weights and personalization (which keeps the separate vertex pass), on RMAT with isolated ids and on a
small graph of dangling and isolated vertices.  The bounds are those of tests/sweep_drivers.py."""
import numpy as np
import pytest

from tests import sweep_drivers as sd

pytestmark = pytest.mark.gpu

SCALE = {"f32w": 16, "f64w": 15, "f32": 16}
LAYOUTS = {**sd.KNOBS, "row-vertex": sd.KNOBS["bands-tail"]}
STEPS = (1, 2, 5, 30)


def graph_for(etype, scale, layout):
    return sd.graph_of(etype, scale, "csr" if layout == "row-vertex" else "csc")


def small_dangling_graph(T):
    """0 -> 1 -> 2 -> 0 (a cycle), 3 -> 1 and 4 -> 1 (sources), 1 -> 5 and 2 -> 6 (sinks), 7 and 8 isolated, a self-loop on 6
    is its only out-edge"""
    s = np.array([0, 1, 2, 3, 4, 1, 2, 6])
    d = np.array([1, 2, 0, 1, 1, 5, 6, 6])
    w = np.linspace(0.5, 1.0, s.size).astype(T)
    return sd.Graph(s, d, 9, T, w, "csc", label=f"dangling-9 {np.dtype(T).name}w")


# ------------------------------------------------------------------------------------------------- fp64 restatement
def _out_weights(graph, out_w=None):
    if out_w is not None:
        ow = np.zeros(graph.V)
        ow[np.asarray(out_w[0])] = np.asarray(out_w[1], graph.T).astype(np.float64)
        return ow
    ow = np.bincount(graph.s, weights=None if graph.w is None else graph.w.astype(np.float64), minlength=graph.V)
    return ow.astype(graph.T).astype(np.float64)   # the driver's sums are rounded to T


def reference_run(graph, alpha, epsilon, max_iterations, guess=None, out_w=None):
    """fp64 PageRank step by step (pagerank_impl.cuh's loop): (states[0..k], diffs, k_ref) as sd.run_until returns them"""
    V = graph.V
    ow = _out_weights(graph, out_w)
    dangling = ow == 0.0
    inv = np.where(dangling, 1.0, 1.0 / np.where(dangling, 1.0, ow))
    At = graph.A   # rows = destinations, fp64 weights

    def step(pr):
        y = alpha * (At @ (pr * inv)) + (alpha * pr[dangling].sum() + 1.0 - alpha) / V
        return y, float(np.abs(y - pr).sum())
    if guess is None:
        x0 = np.full(V, float(graph.T(1) / graph.T(V)))
    else:
        x0 = np.zeros(V)
        x0[np.asarray(guess[0])] = np.asarray(guess[1], graph.T).astype(np.float64)
    return sd.run_until(step, x0, max_iterations, epsilon, max_iterations)


def _rtol(graph, steps, n_pers=0):
    u = sd.unit(graph.T)
    per_step = (sd.sweep_delta(graph.T, int(graph.indeg.max(initial=0))) + 3.0 * u
                + (int(graph.outdeg.max(initial=0)) + graph.V + n_pers) * sd.E + 8.0 * sd.E)
    return sd.SECOND_ORDER * (u + steps * per_step)


def check_epsilon(h, g, graph, epsilon, max_iterations=100, guess=None, out_w=None, alpha=0.85):
    """epsilon > 0: the driver's iteration count, converged flag and values against the restatement"""
    verts, vals, k = sd.pagerank_call(h, g, graph, alpha, epsilon, max_iterations, guess=guess, out_w=out_w)
    xs, diffs, k_ref = reference_run(graph, alpha, epsilon, max_iterations, guess, out_w)
    k_ref = min(k_ref, max_iterations)
    label = f"PageRank {graph.label} epsilon {epsilon:g}"
    # the driver's difference of step j is off by at most the error of the two states it subtracts, summed over V
    tol_diff = [_rtol(graph, j + 2) * (np.abs(xs[j]).sum() + np.abs(xs[j + 1]).sum()) for j in range(len(diffs))]
    sd.check_count(k, k_ref, diffs, epsilon, tol_diff, graph.T, label)
    ref = xs[k]
    got = graph.dense(verts, vals)
    sd.compare(got, ref, _rtol(graph, k), f"{label}, {k} steps", f"pagerank epsilon {np.dtype(graph.T).name}")
    return k


def run_layout(monkeypatch, capfd, graph, layout, steps=STEPS):
    """every PageRank variant on `graph` built under LAYOUTS[layout]"""
    knobs = LAYOUTS[layout]
    capfd.readouterr()
    h, g = graph.create(monkeypatch, knobs)
    for k in steps:
        sd.check_pagerank(h, g, graph, steps=k)
    k = steps[-1]
    rng = np.random.default_rng(5)
    guess = (np.arange(graph.V), rng.uniform(0.0, 2.0 / graph.V, graph.V).astype(graph.T))
    ow = np.bincount(graph.s, weights=None if graph.w is None else graph.w.astype(np.float64), minlength=graph.V)
    out_w = (np.arange(graph.V), (2.0 * ow).astype(graph.T))
    sd.check_pagerank(h, g, graph, steps=k, guess=guess)
    sd.check_pagerank(h, g, graph, steps=k, out_w=out_w)
    sd.check_pagerank(h, g, graph, steps=k, pers=sd.personalizations(graph)["share_with_zeros"], guess=guess)
    eps = 1e-5 if graph.T == np.float32 else 1e-9
    n = check_epsilon(h, g, graph, eps)
    assert 2 < n < 100, f"{graph.label}: converged after {n} steps at epsilon {eps}"
    check_epsilon(h, g, graph, eps, guess=guess, out_w=out_w)
    check_epsilon(h, g, graph, 1e-30, max_iterations=7)   # does not converge: 7 steps, converged = False
    sd.check_layouts(capfd.readouterr().err, graph, knobs, ["pull"], f"pagerank {graph.label} {layout}")


def check_not_converged(h, g, graph):
    """epsilon that no step reaches: max_iterations steps, reported as not converged (cugraph_pagerank raises)"""
    from cugraph_b200 import _capi
    with pytest.raises(_capi.CugraphError) as e:
        sd.pagerank_call(h, g, graph, 0.85, 1e-30, 4, allow_nonconvergence=False)
    assert "PageRank failed to converge." in str(e.value)


def check_launches(h, g, graph):
    """an iteration is the sweep and k_finalize: two launches fewer than a personalized one (k_personalize and
    k_vertex_pass), whatever the layout's sweep launches"""
    pers = sd.personalizations(graph)["share_with_zeros"]

    def per_step(p):
        counts = []
        for k in (3, 4):
            l0 = h.launch_count()
            sd.pagerank_call(h, g, graph, 0.85, 0.0, k, pers=p)
            counts.append(h.launch_count() - l0)
        return counts[1] - counts[0]
    sd.pagerank_call(h, g, graph, 0.85, 0.0, 2)   # layouts and out-weights built
    assert per_step(None) == per_step(pers) - 2


# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("etype", list(SCALE))
@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_pagerank_row_epilogue(monkeypatch, capfd, layout, etype):
    run_layout(monkeypatch, capfd, graph_for(etype, SCALE[etype], layout), layout)


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_pagerank_row_epilogue_launches(monkeypatch, capfd, layout):
    graph = graph_for("f32", SCALE["f32"], layout)
    h, g = graph.create(monkeypatch, LAYOUTS[layout])
    check_launches(h, g, graph)
    check_not_converged(h, g, graph)


@pytest.mark.parametrize("T", [np.float32, np.float64])
def test_pagerank_row_epilogue_dangling(monkeypatch, T):
    graph = small_dangling_graph(T)
    h, g = graph.create(monkeypatch, {})
    for k in (1, 2, 3, 10):
        sd.check_pagerank(h, g, graph, steps=k)
    check_epsilon(h, g, graph, 1e-6 if T == np.float32 else 1e-12)
    sd.check_pagerank(h, g, graph, steps=10, pers=(np.array([5, 7]), np.array([1.0, 3.0], T)))
