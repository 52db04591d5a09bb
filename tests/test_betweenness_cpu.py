"""Betweenness centrality on the CPU: the checks of tests/test_betweenness_gpu.py driven through the Python surface over the
emulation build of the library (tests/emu_py.py), at sizes the emulation runs in seconds; and the oracle of
tests/betweenness_ref.py against networkx on full-source runs."""
import numpy as np
import pytest

from tests import betweenness_ref as ref
from tests import test_betweenness_gpu as t
from tests.emu_py import surface  # noqa: F401


@pytest.mark.parametrize("kind", ["random", "random_sym"])
def test_graphs_emulated(surface, monkeypatch, kind):
    t.check_graph(monkeypatch, kind, 100)


@pytest.mark.parametrize("kind", ["rmat", "rmat_sym"])
def test_rmat_emulated(surface, monkeypatch, kind):
    t.check_graph(monkeypatch, kind, 7, n_sources=(63, 65), full=False)


def test_layouts_emulated(surface, monkeypatch):
    t.check_layouts(monkeypatch, "rmat", 6)
    t.check_layouts(monkeypatch, "rmat_sym", 6)


def test_special_graphs_emulated(surface, monkeypatch):
    t.check_special(monkeypatch)


def test_long_path_emulated(surface):
    t.check_path(500)


def test_diamond_chain_emulated(surface):
    t.check_diamonds()


def test_float64_emulated(surface, monkeypatch):
    t.check_float64(monkeypatch)


def test_bit_identical_repeats_emulated(surface):
    t.check_deterministic("rmat_sym", 8)


def test_errors_emulated(surface):
    t.check_errors()


def test_select_random_vertices_emulated(surface):
    t.check_select_random_vertices()


def test_api_emulated(surface):
    t.check_api()


def test_pylibcugraph_golden_emulated(surface):
    t.check_golden()


@pytest.mark.parametrize("kind", ["random", "random_sym"])
def test_oracle_against_networkx(kind):
    nx = pytest.importorskip("networkx")
    s, d, V, sym = t.edges(kind, 60, 4)
    G = (nx.Graph if sym else nx.DiGraph)()
    G.add_nodes_from(range(V))
    G.add_edges_from(zip(s.tolist(), d.tolist()))
    keep = np.array([G.has_edge(a, b) for a, b in zip(s, d)])
    # networkx counts each vertex pair once: compare on the simple graph (first copy of every edge)
    key = np.asarray(s, np.int64) * V + d
    _, first = np.unique(key, return_index=True)
    first = np.sort(first[(s[first] != d[first]) & keep[first]])
    if sym:
        lo = np.minimum(s, d)[first] * V + np.maximum(s, d)[first]
        _, u = np.unique(lo, return_index=True)
        sel = first[u]
        ss, dd = np.concatenate([s[sel], d[sel]]), np.concatenate([d[sel], s[sel]])
    else:
        ss, dd = s[first], d[first]
    for norm in (False, True):
        for ep in (False, True):
            want = nx.betweenness_centrality(G, normalized=norm, endpoints=ep)
            got = ref.betweenness(ss, dd, V, None, norm, ep, sym, np.float64)
            np.testing.assert_allclose(got, [want[v] for v in range(V)], rtol=1e-9, atol=1e-12)
        want = nx.edge_betweenness_centrality(G, normalized=norm)
        got = ref.edge_betweenness(ss, dd, V, None, norm, sym, np.float64)
        exp = np.array([want[(a, b)] if (a, b) in want else want[(b, a)] for a, b in zip(ss.tolist(), dd.tolist())])
        if sym:  # networkx gives an undirected edge both directions' sum
            got = got[: sel.size] + got[sel.size:]
            exp = exp[: sel.size]
        np.testing.assert_allclose(got, exp, rtol=1e-9, atol=1e-12)
