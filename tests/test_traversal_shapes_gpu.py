"""BFS, SSSP and extract_paths on the graphs and weights that decide their control flow, against the CPU oracle.

RMAT and uniform random graphs are 6-12 BFS levels deep and their weights are U[0,1); the traversal code has branches
that only such inputs never reach.  Here:
- shapes: a long path (natural, random and int64 ids), a grid with edges removed (diameter ~300), a lollipop (an RMAT
  core, a long tail, a clique at its far end: the last BFS levels meet dense rows after the direction-optimising switch
  back), brooms (a hub with k chains whose queue sits at the single-CTA SSSP limits of 2048 entries and 16384 edges for
  many rounds) and a union of small components (multi-source BFS).  Each shape runs symmetric and directed, the directed
  form with store_transposed both ways.
- weights, fp32 and fp64: unit (SSSP distances equal BFS distances), {1, 2, 3} (ties everywhere), all zero and 70 %
  zero (zero-weight plateaus: the predecessor tie passes), log-uniform over 2^-40..2^40 / 2^-300..2^300 (weights absorbed
  by rounding, a window width that means little), subnormals mixed with 1.0, and near-overflow weights around max/8 with
  some max/4, max/2 and one edge of exactly max (a path sum that rounds to inf or to exactly max leaves the vertex
  unreached).
- cutoffs: 0, the smallest weight, exactly a reached distance d* (the comparison is strict: the vertex at d* stays
  unreached), nextafter(d*, inf), a double strictly above d* that rounds down to d* in float, 1e300.
- BFS depth limits 1, D/2, D and D + 1 (D: the depth of the traversal), top-down and direction-optimising.

Distances are bit-exact against the oracle; predecessors pass the oracle's predicates, form a tree (every chain ends at the
source) and, for SSSP, each reached vertex's predecessor edge is tight in the weight type; they are -1 exactly where a
vertex is unreached.  fp32 SSSP with predecessors (the packed distance/predecessor word) and without give the same
distances, and every schedule knob set gives the distances of the default run.

The check_* functions are shared with tests/test_traversal_shapes_cpu.py, which runs them on the CPU emulation of the
library at EMU_SIZES.  Under the emulation this file runs at EMU_SIZES too."""
import collections
import time

import numpy as np
import pytest

import oracle
from oracle.rmat import rmat_edgelist
from tests.test_paths_gpu import (BFS_SCHEDULES, INT_MAX, OFFS64, SSSP_SCHEDULES, _assert_bfs_paths,
                                  _assert_predecessor_tree, _bfs, _bfs_extract_paths, _graph, _sssp)

pytestmark = pytest.mark.gpu

GPU_SIZES = dict(path=10_000, grid=150, core=14, tail=2_000, clique=600, chain=64, components=2_000)
EMU_SIZES = dict(path=160, grid=12, core=8, tail=60, clique=24, chain=3, components=100)
# (name, is_symmetric, store_transposed)
FORMS = (("symmetric", True, False), ("directed", False, False), ("directed-transposed", False, True))
FAMILIES = ("unit", "ints", "zero", "zero70", "loguniform", "subnormal", "overflow")
ALL_SSSP_KNOBS = {"offs64": OFFS64, **SSSP_SCHEDULES}
ALL_BFS_KNOBS = {"offs64": OFFS64, **BFS_SCHEDULES}


def _sizes():
    from cugraph_b200 import _capi
    return EMU_SIZES if _capi.emulated() else GPU_SIZES


# ---------------------------------------------------------------------------------------------------------- shapes
class Shape(collections.namedtuple("Shape", "name s d V ids source_sets")):
    """a directed edge list s -> d over the vertices 0..V-1 (internal indices), the external id of every index, and the
    source sets to traverse from (internal indices)"""

    def edges(self, symmetric):
        return (np.concatenate([self.s, self.d]), np.concatenate([self.d, self.s])) if symmetric else (self.s, self.d)

    def index_of(self, ext):
        """internal index of external ids (-1 stays -1)"""
        ext = np.asarray(ext)
        order = np.argsort(self.ids)
        pos = np.searchsorted(self.ids[order], np.where(ext >= 0, ext, self.ids.min()))
        return np.where(ext >= 0, order[np.clip(pos, 0, self.V - 1)], -1)

    def scatter(self, verts, vals):
        v, x = verts.cpu().numpy(), vals.cpu().numpy()
        out = np.zeros(self.V, dtype=x.dtype)
        out[self.index_of(v)] = x
        return out


def _ids(V, kind, seed):
    if kind == "natural":
        return np.arange(V, dtype=np.int32)
    perm = np.random.default_rng(seed).permutation(V)
    return perm.astype(np.int32) if kind == "random" else (10**12 + 7 * perm).astype(np.int64)


def path(n, ids="natural"):
    s = np.arange(n - 1, dtype=np.int32)
    return Shape(f"path-{n}-{ids}-ids", s, s + 1, n, _ids(n, ids, n), [[0], [n // 2]])


def grid(k, seed=1):
    """k x k grid, edges right and down, about 10 % removed (kept connected enough to have a diameter of about 2k)"""
    v = np.arange(k * k, dtype=np.int32).reshape(k, k)
    s = np.concatenate([v[:, :-1].ravel(), v[:-1, :].ravel()])
    d = np.concatenate([v[:, 1:].ravel(), v[1:, :].ravel()])
    keep = np.random.default_rng(seed).random(s.size) >= 0.1
    return Shape(f"grid-{k}x{k}", s[keep], d[keep], k * k, _ids(k * k, "natural", 0), [[0], [int(v[k // 2, k // 2])]])


def lollipop(scale, tail, clique):
    """an RMAT core, a tail of `tail` vertices from the core's hub, a `clique`-clique at the tail's far end"""
    cs, cd = rmat_edgelist(scale, 16 << scale, seed=40 + scale)
    cs, cd = np.asarray(cs, np.int64), np.asarray(cd, np.int64)
    C = 1 << scale
    hub = int(np.bincount(np.concatenate([cs, cd]), minlength=C).argmax())
    t = np.arange(C, C + tail)
    q = np.arange(C + tail, C + tail + clique)
    qi, qj = np.triu_indices(clique, 1)
    s = np.concatenate([cs, [hub], t[:-1], [t[-1]], q[qi]])
    d = np.concatenate([cd, [t[0]], t[1:], [q[0]], q[qj]])
    V = C + tail + clique
    return Shape(f"lollipop-rmat{scale}-{tail}-{clique}", s.astype(np.int32), d.astype(np.int32), V, _ids(V, "natural", 0),
                 [[hub], [V - 1]])


def broom(k, length):
    """a hub (vertex 0) with k chains of `length` vertices; every chain link is 4 parallel edges, so a chain vertex has
    8 edges in the symmetric form and a queue of k chain vertices holds 8k edges (16384 at k = 2048)"""
    first = 1 + np.arange(k) * length
    s = [np.zeros(k, np.int64)]
    d = [first]
    for i in range(length - 1):
        s.append(first + i)
        d.append(first + i + 1)
    s, d = np.tile(np.concatenate(s), 4), np.tile(np.concatenate(d), 4)
    V = 1 + k * length
    return Shape(f"broom-{k}x{length}", s.astype(np.int32), d.astype(np.int32), V, _ids(V, "natural", 0), [[0]])


def components(n, seed=3):
    """n random components of 3..30 vertices (a random tree plus a few extra edges each); BFS from every other
    component's first vertex at once, and from a single one"""
    r = np.random.default_rng(seed)
    sizes = r.integers(3, 31, n)
    base = np.concatenate([[0], np.cumsum(sizes)[:-1]])
    s, d = [], []
    for b, m in zip(base.tolist(), sizes.tolist()):
        child = np.arange(1, m)
        s.append(b + (r.random(m - 1) * child).astype(np.int64))
        d.append(b + child)
        extra = r.integers(0, m, (2, m // 3))
        s.append(b + extra[0])
        d.append(b + extra[1])
    V = int(sizes.sum())
    return Shape(f"components-{n}", np.concatenate(s).astype(np.int32), np.concatenate(d).astype(np.int32), V,
                 _ids(V, "random", seed), [base[::2].tolist(), [int(base[1])]])


def make_shape(name, sz):
    if name.startswith("broom-"):
        return broom(int(name.split("-")[1]), sz["chain"])
    return {"path": lambda: path(sz["path"]),
            "path-random-ids": lambda: path(sz["path"], "random"),
            "path-int64-ids": lambda: path(sz["path"], "int64"),
            "grid": lambda: grid(sz["grid"]),
            "lollipop": lambda: lollipop(sz["core"], sz["tail"], sz["clique"]),
            "components": lambda: components(sz["components"])}[name]()


# --------------------------------------------------------------------------------------------------------- weights
def weights(family, wd, m, seed):
    r = np.random.default_rng(seed)
    fi = np.finfo(wd)
    if family == "unit":
        return np.ones(m, wd)
    if family == "ints":
        return r.integers(1, 4, m).astype(wd)
    if family == "zero":
        return np.zeros(m, wd)
    if family == "zero70":
        return np.where(r.random(m) < 0.7, 0.0, r.random(m) + 0.01).astype(wd)
    if family == "loguniform":
        e = 40 if wd == np.float32 else 300
        return np.exp2(r.uniform(-e, e, m)).astype(wd)
    if family == "subnormal":
        k = r.integers(1, 2 ** (fi.nmant), m).astype(np.float64)
        sub = np.ldexp(k, fi.minexp - fi.nmant).astype(wd)       # k * the smallest subnormal: exact
        assert (sub < fi.smallest_normal).all() and (sub > 0).all()
        return np.where(r.random(m) < 0.5, wd(1.0), sub).astype(wd)
    if family == "overflow":
        top = fi.max
        u = r.random(m)
        w = np.where(u < 0.2, top / wd(2), np.where(u < 0.4, top / wd(4), (top / wd(8)) * r.uniform(0.5, 1.5, m).astype(wd)))
        w = w.astype(wd)
        w[:2] = top / wd(2)          # on a path: vertex 2 at exactly max from vertex 0
        w[m // 2] = top              # one edge of exactly max
        return w
    raise ValueError(family)


# ------------------------------------------------------------------------------------------------------ SSSP checks
def _cutoffs(ref_d, w, wd):
    """0, the smallest weight, d* (a reached distance), nextafter(d*, inf), for float a double strictly above d* that
    rounds down to d*, 1e300"""
    unreached = np.finfo(wd).max
    reach = np.sort(ref_d[(ref_d > 0) & (ref_d < unreached)])
    out = [("0", 0.0), ("smallest-weight", float(w.min()))]
    if reach.size:
        ds = wd(reach[reach.size // 2])
        out += [("d*", float(ds)), ("nextafter(d*)", float(np.nextafter(ds, wd(np.inf))))]
        if wd == np.float32:
            above = float(ds) + float(np.spacing(ds)) / 4
            assert above > float(ds) and np.float32(above) == ds
            out.append(("double-above-d*", above))
    out.append(("1e300", 1e300))
    return out


def _run_sssp(shape, h, g, src, cutoff=float("inf"), pred=True):
    verts, dist, p = _sssp(h, g, int(shape.ids[src]), cutoff, pred)
    return shape.scatter(verts, dist), (shape.index_of(shape.scatter(verts, p)) if pred else None)


def _assert_sssp(s, d, w, V, src, got_d, got_p, ref_d, case):
    wd = w.dtype.type
    unreached = np.finfo(wd).max
    assert got_d.dtype == wd, case
    bad = np.flatnonzero(got_d.astype(np.float64) != ref_d)
    assert bad.size == 0, f"{case}: {bad.size} distances differ, e.g. vertex {bad[0]}: {got_d[bad[0]]!r} != {ref_d[bad[0]]!r}"
    # the predicate's tolerance is absolute, 1e-6 x the largest weight; one addition rounds by up to half an ulp of the
    # distance, which on a deep fp32 traversal is more than that: allow one ulp of the largest reached distance
    wmax = max(float(w.max()), 1.0)
    rel_tol = max(1e-6, float(np.spacing(got_d[got_d != unreached].max())) / wmax)
    with np.errstate(over="ignore", invalid="ignore"):
        assert oracle.check_sssp_predecessors(s, d, w, V, got_d.astype(np.float64), got_p, src, rel_tol=rel_tol), case
        _assert_predecessor_tree(got_d, got_p, src, unreached)
        # each reached vertex other than the source has a predecessor edge that is tight in the weight type
        tight = (got_p[d] == s) & ((got_d[s] + w).astype(wd) == got_d[d])
    ok = np.zeros(V, bool)
    ok[d[tight]] = True
    ok[src] = True
    assert ok[got_d != unreached].all(), f"{case}: predecessor edge not tight at {np.flatnonzero(~ok & (got_d != unreached))[:5]}"


def check_sssp(monkeypatch, shape, family, wd, knob_sets=ALL_SSSP_KNOBS, cutoffs=True, forms=FORMS):
    """SSSP from every single source of the shape, every form: against the oracle, without predecessors and under every
    cutoff; on the symmetric form also under every knob set"""
    unreached = np.finfo(wd).max
    use_float = wd == np.float32
    for form, sym, st in forms:
        t0 = time.perf_counter()
        s, d = shape.edges(sym)
        w1 = weights(family, wd, shape.s.size, seed=shape.V)
        w = np.concatenate([w1, w1]) if sym else w1
        kw = dict(symmetric=sym, store_transposed=st, vertices=shape.ids, vertex_dtype=shape.ids.dtype, weight_dtype=wd)
        es, ed = shape.ids[s], shape.ids[d]
        h, g = _graph(monkeypatch, {}, es, ed, w, **kw)
        csr = oracle.coo_to_csx(s, d, shape.V, w)
        runs = 0
        for srcs in shape.source_sets:
            if len(srcs) != 1:
                continue
            src = srcs[0]
            case = f"{shape.name} {form} {family} {wd.__name__} source={src}"
            ref_d, _ = oracle.sssp(s, d, w, shape.V, src, use_float=use_float, csr=csr)
            got_d, got_p = _run_sssp(shape, h, g, src)
            _assert_sssp(s, d, w, shape.V, src, got_d, got_p, ref_d, case)
            runs += 1
            if family == "unit":      # SSSP distances are BFS distances, without the oracle
                bd, _ = _run_bfs(shape, h, g, [src], False)
                assert np.array_equal(np.where(bd == INT_MAX, unreached, bd).astype(wd), got_d), case + " against BFS"
            if family == "overflow":  # some vertex with a path from the source is left unreached by overflow
                reach_bfs, _ = oracle.bfs(s, d, shape.V, [src])
                assert ((reach_bfs < INT_MAX) & (ref_d == unreached)).any() or (reach_bfs < INT_MAX).sum() <= 2, case
            if use_float:             # the plain distance word against the packed one
                plain, _ = _run_sssp(shape, h, g, src, pred=False)
                assert np.array_equal(plain, got_d), case + " without predecessors"
                runs += 1
            for kname, knobs in (knob_sets if sym else {}).items():
                hk, gk = _graph(monkeypatch, knobs, es, ed, w, **kw)
                kd, kp = _run_sssp(shape, hk, gk, src)
                assert np.array_equal(kd, got_d), f"{case} knobs={kname}"
                _assert_sssp(s, d, w, shape.V, src, kd, kp, ref_d, f"{case} knobs={kname}")
                runs += 1
            if not cutoffs:
                continue
            for cname, co in _cutoffs(ref_d, w, wd):
                ccase = f"{case} cutoff={cname} ({co!r})"
                ref_c, _ = oracle.sssp(s, d, w, shape.V, src, cutoff=co, use_float=use_float, csr=csr)
                got_c, got_cp = _run_sssp(shape, h, g, src, cutoff=co)
                _assert_sssp(s, d, w, shape.V, src, got_c, got_cp, ref_c, ccase)
                # independently of the oracle: the cut run keeps exactly the distances below the cutoff in weight type
                co_w = np.float64(wd(min(co, float(unreached))))
                want = np.where(ref_d < co_w, ref_d, float(unreached))
                want[src] = 0.0
                assert np.array_equal(got_c.astype(np.float64), want), ccase + " against the uncut run"
                if use_float:
                    plain, _ = _run_sssp(shape, h, g, src, cutoff=co, pred=False)
                    assert np.array_equal(plain, got_c), ccase + " without predecessors"
                runs += 2
        print(f"sssp {shape.name} {form} {family} {wd.__name__}: {runs} runs, {time.perf_counter() - t0:.2f} s")


# ------------------------------------------------------------------------------------------------------- BFS checks
def _run_bfs(shape, h, g, srcs, do, limit=0):
    """BFS distances (int32, INT_MAX where unreached, as the oracle's) and predecessors by internal index.  The
    library returns distances in the vertex type: int64 graphs mark unreached vertices with INT64_MAX"""
    verts, dist, pred = _bfs(h, g, shape.ids[np.asarray(srcs)], do, limit, vertex_dtype=shape.ids.dtype)
    dist = shape.scatter(verts, dist)
    assert dist.dtype == shape.ids.dtype
    dist = np.where(dist == np.iinfo(dist.dtype).max, INT_MAX, dist).astype(np.int32)
    return dist, shape.index_of(shape.scatter(verts, pred))


def check_bfs(monkeypatch, shape, knob_sets=ALL_BFS_KNOBS, depth_limits=True, forms=FORMS):
    """BFS from every source set of the shape, top-down and direction-optimising, every form, with the depth limits
    1, D/2, D, D + 1 and under every knob set"""
    for form, sym, st in forms:
        t0 = time.perf_counter()
        s, d = shape.edges(sym)
        kw = dict(symmetric=sym, store_transposed=st, vertices=shape.ids, vertex_dtype=shape.ids.dtype)
        es, ed = shape.ids[s], shape.ids[d]
        h, g = _graph(monkeypatch, {}, es, ed, **kw)
        knob_graphs = {k: _graph(monkeypatch, v, es, ed, **kw) for k, v in knob_sets.items()}
        csr = oracle.coo_to_csx(s, d, shape.V)
        runs = 0
        for srcs in shape.source_sets:
            ref, _ = oracle.bfs(s, d, shape.V, srcs, csr=csr)
            D = int(ref[ref < INT_MAX].max())
            limits = sorted({0} | ({1, max(D // 2, 1), max(D, 1), D + 1} if depth_limits else set()))
            for do in ((False, True) if sym else (False,)):     # direction-optimising BFS needs a symmetric graph
                case = f"{shape.name} {form} sources={srcs[:4]}{'...' if len(srcs) > 4 else ''} direction_optimizing={do}"
                for limit in limits:
                    lcase = f"{case} depth_limit={limit} (depth {D})"
                    ref_l = ref if limit == 0 else oracle.bfs(s, d, shape.V, srcs, depth_limit=limit, csr=csr)[0]
                    got_d, got_p = _run_bfs(shape, h, g, srcs, do, limit)
                    bad = np.flatnonzero(got_d != ref_l)
                    assert bad.size == 0, f"{lcase}: {bad.size} distances differ, e.g. vertex {bad[0]}: {got_d[bad[0]]} != {ref_l[bad[0]]}"
                    assert oracle.check_bfs_predecessors(s, d, shape.V, got_d, got_p, srcs), lcase
                    if limit:   # independently of the oracle: the limited run is the unlimited one cut at the limit
                        assert np.array_equal(got_d, np.where(ref <= limit, ref, INT_MAX)), lcase + " against the unlimited run"
                    runs += 1
                for kname, (hk, gk) in knob_graphs.items():
                    kd, kp = _run_bfs(shape, hk, gk, srcs, do)
                    assert np.array_equal(kd, ref), f"{case} knobs={kname}"
                    assert oracle.check_bfs_predecessors(s, d, shape.V, kd, kp, srcs), f"{case} knobs={kname}"
                    runs += 1
        print(f"bfs {shape.name} {form}: {runs} runs, {time.perf_counter() - t0:.2f} s")


def check_extract_paths(monkeypatch, shape, forms=FORMS[:2]):
    """extract_paths from the shape's first source to 200 random vertices, the farthest one, an unreached one and the
    source: rows as long as the traversal is deep"""
    assert shape.ids.dtype == np.int32 and np.array_equal(shape.ids, np.arange(shape.V))
    for form, sym, st in forms:
        t0 = time.perf_counter()
        s, d = shape.edges(sym)
        h, g = _graph(monkeypatch, {}, s, d, symmetric=sym, store_transposed=st, vertices=shape.ids)
        source = shape.source_sets[0][0]
        ref, _ = oracle.bfs(s, d, shape.V, [source])
        r = np.random.default_rng(shape.V)
        dests = np.concatenate([r.choice(shape.V, 200), [int(np.where(ref < INT_MAX, ref, -1).argmax())],
                                np.flatnonzero(ref == INT_MAX)[:1], [source]]).astype(np.int32)
        verts, dist, paths = _bfs_extract_paths(h, g, source, dests)
        dist = shape.scatter(verts, dist)
        assert np.array_equal(dist, ref), f"{shape.name} {form}"
        assert paths.shape[1] == 1 + int(ref[ref < INT_MAX].max()), f"{shape.name} {form}"
        _assert_bfs_paths(s, d, shape.V, source, dests, dist, paths)
        print(f"extract_paths {shape.name} {form}: rows of {paths.shape[1]}, {time.perf_counter() - t0:.2f} s")


# =========================================================================================================== tests
BROOMS = ("broom-2047", "broom-2048", "broom-2049", "broom-2100")
BFS_SHAPES = ("path", "path-random-ids", "path-int64-ids", "grid", "lollipop", "components") + BROOMS


@pytest.mark.parametrize("shape", BFS_SHAPES)
def test_bfs_shapes(monkeypatch, shape):
    big = shape in ("lollipop",) + BROOMS
    check_bfs(monkeypatch, make_shape(shape, _sizes()), knob_sets={"offs64": OFFS64} if big else ALL_BFS_KNOBS)


@pytest.mark.parametrize("shape", ["path", "grid", "lollipop"])
def test_extract_paths_shapes(monkeypatch, shape):
    check_extract_paths(monkeypatch, make_shape(shape, _sizes()))


# the full knob and cutoff sets on the path and the grid; the larger shapes with a subset
SSSP_CASES = ([(sh, fam, True, True) for sh in ("path", "grid") for fam in FAMILIES]
              + [(sh, fam, False, True) for sh in ("path-random-ids", "path-int64-ids") for fam in FAMILIES]
              + [("lollipop", fam, False, False) for fam in FAMILIES]
              + [(b, fam, False, False) for b in BROOMS for fam in ("unit", "ints", "zero70")])
SUBSET = {k: ALL_SSSP_KNOBS[k] for k in ("offs64", "no-single-cta-rounds", "not-adaptive")}


@pytest.mark.parametrize("wdtype", [np.float32, np.float64])
@pytest.mark.parametrize("shape,family,all_knobs,cutoffs", SSSP_CASES, ids=[f"{c[0]}-{c[1]}" for c in SSSP_CASES])
def test_sssp_shapes(monkeypatch, shape, family, all_knobs, cutoffs, wdtype):
    sh = make_shape(shape, _sizes())
    forms = FORMS if not shape.startswith("broom") or family == "unit" else FORMS[:1]
    check_sssp(monkeypatch, sh, family, wdtype, knob_sets=ALL_SSSP_KNOBS if all_knobs else SUBSET, cutoffs=cutoffs, forms=forms)
