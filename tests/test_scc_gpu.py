"""Strongly connected components on the GPU (cugraph_strongly_connected_components through the pylibcugraph-compatible
wrapper) against tests/scc_ref.py's scc, the restatement of the reference test's Tarjan (strongly_connected_components_test.cpp),
with scipy's connected_components(connection="strong") as a second check on the large graphs.

What is checked of every result: the partition equals the oracle's, every label is the id of a member of its own component,
and the labels do not change from one call to the next.  The shapes that stress one phase each: a directed chain (resolved
by the trim alone), one directed cycle (one SCC, the forward and backward reaches are as deep as the cycle is long) and a
chain of small cycles joined one way (the colouring rounds).

The check_* functions are shared with tests/test_scc_cpu.py, which runs them on the CPU emulation of the library at
smaller sizes."""
import json
import os

import numpy as np
import pytest

from oracle.rmat import rmat_edgelist
from tests.gpu_util import make_graph
from tests.scc_ref import scc as scc_ref

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OFFS64 = {"OFFS64_MIN_EDGES": "0"}


def golden_cases():
    with open(os.path.join(ROOT, "tests", "golden", "scc_golden.json")) as f:
        return json.load(f)["cases"]


def scc(h, g):
    from cugraph_b200 import pylibcugraph as plc
    verts, labels = plc.strongly_connected_components(h, g, None, None, None, None, False)
    return verts.cpu().numpy(), labels.cpu().numpy()


def _graph(monkeypatch, knobs, *args, **kw):
    """make_graph with CUGRAPH_B200_<knob> set while its handle is created (the handle reads the knobs once)"""
    for k, v in knobs.items():
        monkeypatch.setenv("CUGRAPH_B200_" + k, v)
    try:
        return make_graph(*args, **kw)
    finally:
        for k in knobs:
            monkeypatch.delenv("CUGRAPH_B200_" + k)


def assert_partition(ids, verts, labels, ref):
    """(verts, labels) in external ids against ref, a component index per vertex of `ids` (ascending external ids):
    the same partition, and the label of every vertex is a member of its own component"""
    assert verts.size == ids.size and np.array_equal(np.sort(verts), ids)
    pos = np.searchsorted(ids, verts)
    comp = ref[pos]
    lab_pos = np.searchsorted(ids, labels)
    assert np.all(lab_pos < ids.size) and np.array_equal(ids[np.minimum(lab_pos, ids.size - 1)], labels), "a label is not a vertex"
    assert np.array_equal(ref[lab_pos], comp), "a label is not a member of its vertex's component"
    # members of one component share one label: with the line above, the partitions are equal
    n_comp = len(np.unique(ref))
    assert len(np.unique(labels)) == n_comp
    assert len(set(zip(comp.tolist(), labels.tolist()))) == n_comp


def dense(src, dst, vertices=None):
    parts = [src, dst] + ([vertices] if vertices is not None else [])
    ids, inv = np.unique(np.concatenate(parts), return_inverse=True)
    return ids, inv[:len(src)], inv[len(src):len(src) + len(dst)]


def check_edges(monkeypatch, src, dst, knobs=None, scipy_check=False, repeat=True, **kw):
    """SCC of the directed edge list against the oracle; returns (verts, labels)"""
    src, dst = np.asarray(src), np.asarray(dst)
    h, g = _graph(monkeypatch, knobs or {}, src, dst, **kw)
    verts, labels = scc(h, g)
    ids, s, d = dense(src, dst, kw.get("vertices"))
    ref = scc_ref(s, d, ids.size)
    assert_partition(ids, verts, labels, ref)
    if scipy_check:
        import scipy.sparse as sp
        from scipy.sparse.csgraph import connected_components
        n, lab = connected_components(sp.coo_matrix((np.ones(s.size), (s, d)), shape=(ids.size, ids.size)).tocsr(),
                                      directed=True, connection="strong")
        assert n == len(np.unique(ref)) and len(set(zip(ref.tolist(), lab.tolist()))) == n
    if repeat:
        v2, l2 = scc(h, g)
        assert np.array_equal(v2, verts) and np.array_equal(l2, labels), "a second call changed the labels"
    return verts, labels


def check_goldens(monkeypatch):
    for name, c in golden_cases().items():
        verts, labels = check_edges(monkeypatch, np.asarray(c["src"], np.int32), np.asarray(c["dst"], np.int32),
                                    scipy_check=True)
        if "scc_comp_vertices" in c:  # the reference test's own expectation (ids 0 .. n-1)
            got = {}
            for v, lab in zip(verts.tolist(), labels.tolist()):
                got.setdefault(lab, []).append(v)
            assert sorted(sorted(m) for m in got.values()) == sorted(c["scc_comp_vertices"]), name


def check_legacy_csr(c):
    """the reference test's form: CSR arrays and a labels array written in place (strongly_connected_components.pyx)"""
    import scipy.sparse as sp
    import torch
    from cugraph_b200 import pylibcugraph as plc
    nv = c["num_vertices"]
    csr = sp.coo_matrix((np.ones(len(c["src"]), np.float32), (c["src"], c["dst"])), shape=(nv, nv)).tocsr()
    offs = torch.as_tensor(csr.indptr.astype(np.int32)).cuda()
    idx = torch.as_tensor(csr.indices.astype(np.int32)).cuda()
    w = torch.as_tensor(csr.data.astype(np.float32)).cuda()
    labels = torch.zeros(nv, dtype=torch.int32).cuda()
    assert plc.strongly_connected_components(None, None, offs, idx, w, labels, False) is None
    got = {}
    for v, lab in enumerate(labels.cpu().numpy().tolist()):
        got.setdefault(lab, []).append(v)
    assert sorted(sorted(m) for m in got.values()) == sorted(c["scc_comp_vertices"])


def check_random(monkeypatch, V, E, seed, knobs=None):
    """directed graphs with hubs on both sides, multi-edges and self-loops; both storage orientations give one partition"""
    from tests.test_emu_staging_cpu import make_edges
    s, d, _ = make_edges(V, E, seed=seed, id_offset=3)
    _, l0 = check_edges(monkeypatch, s, d, knobs, store_transposed=False)
    check_edges(monkeypatch, s, d, knobs, store_transposed=True, repeat=False)
    return l0


def check_loops_and_multi_edges(monkeypatch, V, E, seed):
    """self-loops and repeated edges change no component"""
    r = np.random.default_rng(seed)
    s, d = r.integers(0, V, E).astype(np.int32), r.integers(0, V, E).astype(np.int32)
    keep = s != d
    s, d = s[keep], d[keep]
    ids, si, di = dense(s, d)
    ref = scc_ref(si, di, ids.size)
    loops = r.choice(ids, size=max(1, ids.size // 4), replace=False).astype(np.int32)
    dup = r.integers(0, s.size, s.size // 3)
    s2, d2 = np.concatenate([s, loops, s[dup], s]), np.concatenate([d, loops, d[dup], d])
    h, g = _graph(monkeypatch, {}, s2, d2)
    assert_partition(ids, *scc(h, g), ref)


def check_both_directions_equals_wcc(monkeypatch, V, E, seed):
    """every edge given in both directions: SCC of the directed graph is WCC of the symmetric one, labels included (the
    same rule over the same internal numbering)"""
    from cugraph_b200 import pylibcugraph as plc
    r = np.random.default_rng(seed)
    a, b = r.integers(0, V, E).astype(np.int32), r.integers(0, V, E).astype(np.int32)
    s, d = np.concatenate([a, b]), np.concatenate([b, a])
    h, g = _graph(monkeypatch, {}, s, d)
    verts, labels = scc(h, g)
    hw, gw = _graph(monkeypatch, {}, s, d, symmetric=True)
    wv, wl = plc.weakly_connected_components(hw, gw, None, None, None, None, False)
    assert np.array_equal(verts, wv.cpu().numpy()) and np.array_equal(labels, wl.cpu().numpy())


def check_symmetric_rejected(monkeypatch):
    from cugraph_b200 import _capi
    h, g = _graph(monkeypatch, {}, np.array([0, 1], np.int32), np.array([1, 0], np.int32), symmetric=True)
    with pytest.raises(_capi.CugraphRuntimeError, match="weakly_connected_components"):
        scc(h, g)


def check_empty_and_isolated(monkeypatch):
    e = np.zeros(0, np.int32)
    h, g = _graph(monkeypatch, {}, e, e)
    verts, labels = scc(h, g)
    assert verts.size == 0 and labels.size == 0
    # isolated vertices from the vertex list are singletons; so are vertices of an edgeless graph
    s, d = np.array([10, 11, 12, 13], np.int32), np.array([11, 12, 10, 10], np.int32)
    check_edges(monkeypatch, s, d, vertices=np.array([10, 11, 12, 13, 40, 7], np.int32))
    check_edges(monkeypatch, e, e, vertices=np.array([5, 3, 9], np.int32))


def check_int64_renumber_false(monkeypatch, V, E, seed, knobs=None):
    """64-bit external ids, and renumber=False (results in vertex order, ids as given)"""
    from tests.test_emu_staging_cpu import make_edges
    s, d, _ = make_edges(V, E, seed=seed)
    big = 5_000_000_000
    verts, labels = check_edges(monkeypatch, s.astype(np.int64) * 7 + big, d.astype(np.int64) * 7 + big, knobs,
                                vertex_dtype=np.int64)
    assert verts.dtype == np.int64 and labels.dtype == np.int64
    vs = np.arange(V, dtype=np.int32)
    verts, labels = check_edges(monkeypatch, s, d, knobs, renumber=False, vertices=vs)
    assert np.array_equal(verts, vs)


def chain(n):
    p = np.random.default_rng(n).permutation(n).astype(np.int32)  # ids carry no order
    return p[:-1], p[1:]


def cycle(n):
    s, d = chain(n)
    return np.append(s, d[-1]), np.append(d, s[0])


def cycle_chain(n_cycles, k):
    """n_cycles directed cycles of k vertices, cycle i joined to cycle i + 1 by one edge"""
    base = np.arange(n_cycles, dtype=np.int64)[:, None] * k
    ring = np.arange(k)
    s = (base + ring).ravel()
    d = (base + (ring + 1) % k).ravel()
    s = np.concatenate([s, base[:-1, 0] + k // 2])
    d = np.concatenate([d, base[1:, 0]])
    p = np.random.default_rng(k).permutation(n_cycles * k)
    return p[s].astype(np.int32), p[d].astype(np.int32)


def check_shapes(monkeypatch, n, n_cycles, k, knobs=None):
    for s, d in (chain(n), cycle(n), cycle_chain(n_cycles, k)):
        check_edges(monkeypatch, s, d, knobs, repeat=False)


def check_api():
    """cugraph-style layer: a directed Graph gives 'vertex' / 'labels'; an undirected (symmetric) one is rejected"""
    import pandas as pd
    from cugraph_b200 import _capi, api
    s, d = cycle_chain(20, 3)
    df = pd.DataFrame({"src": s, "dst": d})
    G = api.Graph(directed=True).from_pandas_edgelist(df, source="src", destination="dst")
    out = api.strongly_connected_components(G)
    assert list(out.columns) == ["vertex", "labels"]
    ids, si, di = dense(s, d)
    assert_partition(ids, out["vertex"].to_numpy(), out["labels"].to_numpy(), scc_ref(si, di, ids.size))
    GU = api.Graph(directed=False).from_pandas_edgelist(df, source="src", destination="dst")
    with pytest.raises(_capi.CugraphRuntimeError, match="weakly_connected_components"):
        api.strongly_connected_components(GU)


def check_rmat(monkeypatch, scale, seed, knobs=None):
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed)
    check_edges(monkeypatch, np.asarray(s, np.int32), np.asarray(d, np.int32), knobs, scipy_check=True)
    return s, d


def run_reference_c_test(suffix):
    import subprocess
    exe = os.path.join(ROOT, "oracle", "_ref", f"ref_strongly_connected_components_test{suffix}")
    if not os.path.exists(exe):
        pytest.skip("oracle/_ref/ref_strongly_connected_components_test* not built (needs the reference sources at build time)")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RUNNING:")]
    assert len(lines) == 1, r.stdout
    assert lines[0].startswith("RUNNING: test_strongly_connected_components...") and lines[0].endswith("- passed"), r.stdout
    assert "ASSERTION FAILED" not in r.stdout


# ---- on the GPU
def test_scc_goldens_gpu(monkeypatch):
    check_goldens(monkeypatch)
    for name, c in golden_cases().items():
        if "scc_comp_vertices" in c:
            check_legacy_csr(c)


@pytest.mark.parametrize("scale", [16, 18])
def test_scc_rmat_gpu(monkeypatch, scale):
    check_rmat(monkeypatch, scale, seed=scale)


def test_scc_rmat_scrambled_int64_and_renumber_false_gpu(monkeypatch):
    s, d = rmat_edgelist(16, 16 << 16, seed=7)
    s, d = np.asarray(s, np.int64), np.asarray(d, np.int64)
    perm = np.random.default_rng(7).permutation(1 << 16).astype(np.int64) * 131 + 3_000_000_000
    check_edges(monkeypatch, perm[s], perm[d], vertex_dtype=np.int64, repeat=False)
    check_edges(monkeypatch, s.astype(np.int32), d.astype(np.int32), renumber=False,
                vertices=np.arange(1 << 16, dtype=np.int32), store_transposed=True, repeat=False)


def test_scc_random_both_orientations_gpu(monkeypatch):
    check_random(monkeypatch, 200_000, 1_000_000, seed=5)


def test_scc_offs64_gpu(monkeypatch):
    check_random(monkeypatch, 50_000, 400_000, seed=6, knobs=OFFS64)
    check_rmat(monkeypatch, 16, seed=8, knobs=OFFS64)


def test_scc_loops_multi_edges_and_wcc_gpu(monkeypatch):
    check_loops_and_multi_edges(monkeypatch, 100_000, 300_000, seed=9)
    check_both_directions_equals_wcc(monkeypatch, 100_000, 150_000, seed=10)


def test_scc_inputs_gpu(monkeypatch):
    check_symmetric_rejected(monkeypatch)
    check_empty_and_isolated(monkeypatch)
    check_int64_renumber_false(monkeypatch, 100_000, 500_000, seed=11)


def test_scc_phase_shapes_gpu(monkeypatch):
    check_shapes(monkeypatch, 100_000, 200, 5)


def test_scc_api_gpu():
    check_api()


def test_reference_scc_c_test_gpu():
    run_reference_c_test("_gpu")
