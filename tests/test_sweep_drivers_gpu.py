"""Katz, eigenvector centrality, HITS and personalized PageRank on the H100, step for step against fp64 references
(tests/sweep_drivers.py), on every sweep layout: the plain sweep, the piece stream, the piece stream in bands with a tail,
and 64-bit offsets.  float32 weights on directed RMAT-16 and float64 on RMAT-15 (the x vector spans more than one 192 KiB
shared-memory slice of either width), and unweighted RMAT-16; multi-edges, self-loops and isolated ids kept.  Then the
other orientations (the re-sorted pull view of a CSR graph, a symmetric graph, CSR input), scattered int64 ids, one graph
through many calls, edge cases, and PageRank's expensive input checks.  The worst observed / bound per algorithm and type is
printed at the end of the module."""

import numpy as np
import pytest

from tests import sweep_drivers as sd

pytestmark = pytest.mark.gpu

SCALE = {"f32w": 16, "f64w": 15, "f32": 16}
ALGORITHMS = ["katz", "eigenvector", "hits", "personalized"]


@pytest.fixture(scope="module", autouse=True)
def report_margins(request):
    """the margins on record: printed past pytest's output capture when the module is done"""
    yield
    capman = request.config.pluginmanager.getplugin("capturemanager")
    if sd.WORST and capman is not None:
        with capman.global_and_fixture_disabled():
            print("\nworst |got - ref| / bound per algorithm and element type:")
            for k in sorted(sd.WORST):
                print(f"  {k:<40} {sd.WORST[k]:.3e}")


def _graph(etype, orientation="csc", scattered_ids=False):
    return sd.graph_of(etype, SCALE[etype], orientation, scattered_ids)


@pytest.mark.parametrize("etype", list(SCALE))
@pytest.mark.parametrize("layout", list(sd.KNOBS))
@pytest.mark.parametrize("algorithm", ALGORITHMS)
def test_driver_layouts(monkeypatch, capfd, algorithm, layout, etype):
    sd.run_case(algorithm, monkeypatch, capfd, _graph(etype), layout)


@pytest.mark.parametrize("orientation", ["csr", "symmetric", "csr-input"])
@pytest.mark.parametrize("layout", ["stream", "bands-tail"])
@pytest.mark.parametrize("algorithm", ALGORITHMS)
def test_driver_orientations(monkeypatch, capfd, algorithm, layout, orientation):
    """store_transposed=False (the re-sorted pull view; HITS sweeps the stored CSR), a symmetric graph (one view for both
    sides of HITS) and a graph given as CSR arrays"""
    sd.run_case(algorithm, monkeypatch, capfd, _graph("f32w", orientation), layout)


@pytest.mark.parametrize("algorithm", ALGORITHMS)
def test_driver_scattered_int64_ids(monkeypatch, capfd, algorithm):
    sd.run_case(algorithm, monkeypatch, capfd, _graph("f64w", "csr", scattered_ids=True), "bands-tail")


@pytest.mark.parametrize("layout,orientation", [(lay, "csc") for lay in sd.KNOBS] + [("bands-tail", "csr")])
def test_one_graph_many_calls(monkeypatch, capfd, layout, orientation):
    sd.run_many_calls(monkeypatch, capfd, _graph("f32w", orientation), layout)


# ---------------------------------------------------------------------------------------------------------- edge cases
def test_isolated_vertices_only(monkeypatch, capfd):
    """no edges: Katz and eigenvector give 1/sqrt(V) after two steps; HITS finds no positive norm"""
    from cugraph_b200 import _capi
    V = 37
    for T in (np.float32, np.float64):
        graph = sd.Graph(np.zeros(0, np.int64), np.zeros(0, np.int64), V, T, np.zeros(0, T), "csc", label="isolated")
        h, g = graph.create(monkeypatch, {})
        sd.check_katz(h, g, graph, 0.5, 1.0, 1e-3)
        sd.check_eigenvector(h, g, graph, 1e-6)
        verts, vals, k = sd.centrality_call("katz_centrality", h, g, None, 0.5, 1.0, 1e-3, 100, 0)
        assert k == 2 and np.allclose(vals.cpu().numpy(), 1.0 / np.sqrt(V), rtol=4 * sd.unit(T), atol=0)
        verts, vals, k = sd.centrality_call("eigenvector_centrality", h, g, 1e-6, 100, 0)
        assert k == 2 and np.allclose(vals.cpu().numpy(), 1.0 / np.sqrt(V), rtol=4 * sd.unit(T), atol=0)
        with pytest.raises(_capi.CugraphError) as e:
            sd.hits_call(h, g, 1e-6, 100)
        assert e.value.code == _capi.UNKNOWN_ERROR and "Norm is required to be a positive value." in str(e.value)


def test_single_self_loop(monkeypatch, capfd):
    for T in (np.float32, np.float64):
        graph = sd.Graph(np.array([0]), np.array([0]), 1, T, np.array([0.75], T), "csc", label="self-loop")
        h, g = graph.create(monkeypatch, {})
        sd.check_katz(h, g, graph, 0.5, 1.0, 1e-6)
        sd.check_eigenvector(h, g, graph, 1e-6)
        sd.check_hits(h, g, graph, 1e-6)
        sd.check_pagerank(h, g, graph, steps=5)
        sd.check_pagerank(h, g, graph, steps=5, pers=(np.array([0]), np.array([2.0], T)))


def test_too_few_iterations(monkeypatch, capfd):
    """each driver stops with its "failed to converge" error when max_iterations is below the step it would converge at"""
    from cugraph_b200 import _capi
    graph = _graph("f32w")
    h, g = graph.create(monkeypatch, {})
    eps = sd.epsilons(graph)
    calls = {"Katz Centrality failed to converge.":
             lambda: sd.centrality_call("katz_centrality", h, g, None, sd.katz_alpha(graph), 1.0, eps["katz"], 2, 0),
             "Eigenvector Centrality failed to converge.":
             lambda: sd.centrality_call("eigenvector_centrality", h, g, eps["eigenvector"], 2, 0),
             "HITS failed to converge.": lambda: sd.hits_call(h, g, eps["hits"], 2),
             "PageRank failed to converge.":
             lambda: sd.pagerank_call(h, g, graph, 0.85, 1e-9, 3, allow_nonconvergence=False)}
    for message, call in calls.items():
        with pytest.raises(_capi.CugraphError) as e:
            call()
        assert e.value.code == _capi.UNKNOWN_ERROR and message in str(e.value), str(e.value)


# ------------------------------------------------------------------------------------- PageRank's expensive input checks
def _small(T=np.float32):
    return sd.rmat(10, 77, T, True, "csc")


def _out_weights(graph):
    ow = np.bincount(graph.s, weights=graph.w.astype(np.float64), minlength=graph.V)
    return np.arange(graph.V), ow.astype(graph.T)


def _expect(code, message, call):
    from cugraph_b200 import _capi
    with pytest.raises(_capi.CugraphError) as e:
        call()
    assert e.value.code == code and message in str(e.value), str(e.value)


@pytest.mark.parametrize("T", [np.float32, np.float64])
def test_pagerank_expensive_checks(monkeypatch, T):
    """with do_expensive_check: negative precomputed out-weight sums, negative personalization values and repeated
    personalization vertices are rejected with the reference's messages (pagerank_impl.cuh:90-175)"""
    from cugraph_b200 import _capi
    graph = _small(T)
    h, g = graph.create(monkeypatch, {})
    ids, ow = _out_weights(graph)
    neg_ow = ow.copy()
    neg_ow[5] = -1.0
    pers = sd.personalizations(graph)["share_with_zeros"]
    neg = (pers[0], pers[1].copy())
    neg[1][1] = -0.5
    dup = (np.concatenate([pers[0], pers[0][:1]]), np.concatenate([pers[1], pers[1][:1]]))
    U = _capi.UNKNOWN_ERROR
    _expect(U, "Invalid input argument: outgoing edge weight sum values should be non-negative.",
            lambda: sd.pagerank_call(h, g, graph, 0.85, 0.0, 5, out_w=(ids, neg_ow), expensive=True))
    _expect(U, "Invalid input argument: peresonalization values should be non-negative.",
            lambda: sd.pagerank_call(h, g, graph, 0.85, 0.0, 5, pers=neg, expensive=True))
    _expect(U, "Invalid input argument: personalization vertices should not contain duplicate entries.",
            lambda: sd.pagerank_call(h, g, graph, 0.85, 0.0, 5, pers=dup, expensive=True))
    # the same calls without the check are not rejected (nothing is checked, as in the reference)
    sd.pagerank_call(h, g, graph, 0.85, 0.0, 5, out_w=(ids, neg_ow))
    sd.pagerank_call(h, g, graph, 0.85, 0.0, 5, pers=neg)


@pytest.mark.parametrize("T", [np.float32, np.float64])
def test_pagerank_expensive_checks_pass_valid_inputs(monkeypatch, T):
    """valid inputs give the reference's values with and without the check; without it the driver launches exactly the
    kernels it launched before these checks existed: the checks' own launches are the only difference (the edge weights:
    one count, as before; out-weights: one count; personalization: one count, a 4-launch sort, one scan for repeats)"""
    graph = _small(T)
    h, g = graph.create(monkeypatch, {})
    ids, ow = _out_weights(graph)
    pers = sd.personalizations(graph)["share_with_zeros"]
    steps = 7
    sd.pagerank_call(h, g, graph, 0.85, 0.0, steps)     # the layout and the cached out-weight sums
    launches = {}
    for expensive in (False, True, False):
        for what, kw in (("pers", dict(pers=pers)), ("out_w", dict(out_w=(ids, ow))), ("both", dict(pers=pers, out_w=(ids, ow)))):
            l0 = h.launch_count()
            verts, vals, k = sd.pagerank_call(h, g, graph, 0.85, 0.0, steps, expensive=expensive, **kw)
            launches.setdefault((what, expensive), set()).add(h.launch_count() - l0)
            assert k == steps
    sd.check_pagerank(h, g, graph, steps=steps, pers=pers)
    sd.check_pagerank(h, g, graph, steps=steps, pers=pers, out_w=(ids, ow))
    plain = {w: launches[(w, False)] for w in ("pers", "out_w", "both")}
    assert all(len(v) == 1 for v in plain.values()), plain
    extra = {"pers": 1 + 6, "out_w": 1 + 1, "both": 1 + 7}
    for w, n in extra.items():
        assert launches[(w, True)] == {next(iter(plain[w])) + n}, (w, launches)
