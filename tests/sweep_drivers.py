"""The single-GPU drivers of the pull sweep — Katz, eigenvector centrality, HITS and (personalized) PageRank — checked step
for step against fp64 references: the harness of tests/test_sweep_drivers_gpu.py (the H100) and
tests/test_sweep_drivers_cpu.py (the emulation build of the library, tests/emu_py.py).

Each check calls the C entry point, reads the iteration count k the driver reports, and runs its fp64 reference for exactly
k steps (check_*: the call; verify_*: the check of a result by internal id, which the multi-GPU harness shares).  k itself
must be the step at which the reference converges under the driver's own test (Katz: diff < epsilon; eigenvector, HITS:
diff < V epsilon, the threshold formed in T as the driver forms it).  The two may differ by one step only
where the reference's difference at the earlier of the two steps lies within the bound below of the threshold; in float64
that bound is ~1e-12 of the threshold, so there the counts must agree.  HITS' hub_score_differences must match the
reference's last difference within the same bound.

The bound.  Every driver iterates a non-negative map (weights and values are non-negative, alpha >= 0).  With u = u_T
(2^-24 for float32, 2^-53 for float64), e = 2^-53 and d_max the most entries of a row of the swept view:

- One sweep.  tests/sweep_rows.py bounds a row by |y - y*| <= 2 (S (4u + d 2^-52) + u |y*|) with S = alpha |A| |x|; here
  S <= |y*| (every term is non-negative, and the constant term the sweep adds is too), so a sweep adds at most
      delta = 2 (5u + d_max 2^-52)
  of componentwise relative error.
- A vector pass adds its roundings: a scaling (T)((double)v * (1/s)) u + 2e, the eigenvector add y + x u, PageRank's x = pr / out_w u.
  An fp64 sum of n non-negative terms (norms, maxima are exact, differences, the dangling sum, the personalization sum) is
  off by at most n e relatively, in any order of the atomics.
- Propagation.  A non-negative linear map does not expand the componentwise relative error of its input, nor does adding a
  non-negative constant (Katz' beta, PageRank's unvarying term and personalization).  Where the drivers normalise (the
  eigenvector's L2 norm, HITS' maxima), the same holds in Hilbert's projective metric d_H, which a normalisation does not
  change; a componentwise relative perturbation r adds at most 2r to d_H.  So errors grow at most linearly in k:
      Katz         e_k <= delta * min(k, 1 / (1 - rho)),  rho = alpha ||A||_inf < 1: the constant beta takes the share
                   (alpha A x)_i / (alpha A x + beta)_i <= rho of each row, so the error contracts by rho per step;
                   the final L2 normalisation doubles it and adds V e + u + 2e.
      eigenvector  D_k <= 2k (delta + 2u + 2e); the result, of norm 1 + theta (|theta| <= V e + u + 2e), is off by at most
                   expm1(D_k) + theta componentwise.
      HITS         D_k <= D_0 + 2k (delta_in + delta_out + u + 2e), D_0 = 2(u + 2e) for an initial guess (the driver
                   divides it by its sum) and 0 otherwise; authorities D_{k-1} + 2(delta_in + u + 2e); expm1 of that,
                   plus V e + u + 2e with normalize (a second division, by the sum).
      PageRank     e_k <= u + k (delta + 3u + (d_max_out + V + n_pers) e + 8e): the start (T)(1/V), per step the sweep, x
                   = pr / out_w, the out-weight sums rounded to T, the dangling and personalization sums, the
                   personalization's own rounding into y.
  The observed error sits orders of magnitude below these bounds; a bound of a few units of u per step is what lets the
  checks see a dropped edge, a stale maximum or a misplaced addition (1e-4 relative and less).  Second-order terms are
  covered by the factor SECOND_ORDER.
- Exact zeros: where the reference is 0 (the hubs of a vertex without out-edges, the authorities of one without in-edges,
  personalized scores of vertices nothing reaches) the driver must give exactly 0.

The multi-GPU drivers (cugraph_b200/mg.py, checked by tests/mg_sweep_drivers.py) run the same steps with the sweep spread
over an R x C grid: x is all-gathered, every block sweeps its rows, and the partial y are reduce-scattered over a group of
G members (the row group, G = C, for the pull sweep; the column group, G = R, for HITS' transposed sweep).
- The all-gather copies: x is exact.
- A block's row holds a subset of the graph row's entries, at most d_max of them, and every term is non-negative, so the
  block's partial y is within sweep_delta(T, d_max) of its own exact value, relatively (the bound above, rounded to T).
- The reduce-scatter adds G non-negative values in T: G - 1 roundings, each relative to a partial sum no larger than the
  total, whatever the order (NCCL's ring and the in-process stand-in alike).  So one sweep adds at most
      delta_G = sweep_delta(T, d_max) + (G - 1) u,
  which the verifiers take as extra = (G - 1) u on top of delta; HITS takes one for each of its two sweeps.
- Out-weight sums: fp64 sums over the blocks, reduce-scattered in fp64 and rounded once to T: one summation tree of the
  vertex's out-weights, at most d_max_out - 1 fp64 additions, as on one GPU.  The owner steps' partials (norms,
  differences, the dangling sum) are fp64 sums of non-negative terms all-reduced in fp64: within n e.  Maxima are exact.
So every bound above holds with delta_G in place of delta, and nothing else changes.

The worst |got - ref| / (rtol |ref|) of each check is returned, recorded in WORST, printed with -s, and quoted with the
bound in any failure message.

CUGRAPH_B200_BUILD_TRACE=1 makes the layout builder print the shape of each piece stream it builds; every check asserts
that the layouts built for the views it swept are the ones its knobs ask for (tests/sweep_rows.py: expected_layout,
check_trace)."""
import collections
import ctypes as C
import math
import re

import numpy as np

from tests import sweep_rows as sr

E = 2.0 ** -53
SECOND_ORDER = 1.01
EMULATED_MAX_SCALE = 10
EMU_L2 = 1 << 20                 # the emulated device's L2 (emu/cuda_runtime.h)
KNOBS = {"plain": {"SWEEP_MIN_EDGES": 1 << 40},
         "stream": {"SWEEP_MIN_EDGES": 0},
         "bands-tail": {"SWEEP_MIN_EDGES": 0, "SWEEP_BANDS": 3, "SWEEP_TAIL_DEGREE": 8},
         "offs64": {"OFFS64_MIN_EDGES": 0}}
WORST = collections.defaultdict(float)


def unit(T):
    return 2.0 ** -53 if T == np.float64 else 2.0 ** -24


def sweep_delta(T, d_max):
    return 2.0 * (5.0 * unit(T) + d_max * 2.0 ** -52)


def emulated():
    from cugraph_b200 import _capi
    return _capi.emulated()


def scale_of(scale):
    return min(scale, EMULATED_MAX_SCALE) if emulated() else scale


def l2_bytes():
    if emulated():
        return EMU_L2
    import torch
    return int(torch.cuda.get_device_properties(0).L2_cache_size)


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
class Graph:
    """an edge list over internal ids 0..V-1 (multi-edges and self-loops kept), its fp64 matrices and how the library is
    given it: orientation ("csc": store_transposed, "csr", "symmetric", "csr-input"), weights in T or none, external ids
    (the identity, or scattered int64 ids)"""

    def __init__(self, s, d, V, T=np.float32, w=None, orientation="csc", ids=None, label=""):
        import scipy.sparse as sp
        self.s, self.d, self.V, self.T, self.orientation, self.ids = s, d, V, T, orientation, ids
        self.w = None if w is None else np.asarray(w, T)
        self.label = label
        w64 = np.ones(s.size) if self.w is None else self.w.astype(np.float64)
        self.A = sp.csr_matrix((w64, (d.astype(np.int64), s.astype(np.int64))), shape=(V, V))    # pulled: rows = destinations
        self.A.sum_duplicates()
        self.N = sp.csr_matrix((np.ones(s.size), (d.astype(np.int64), s.astype(np.int64))), shape=(V, V))   # unweighted
        self.N.sum_duplicates()
        self.Nt = self.N.T.tocsr()
        self.indeg = np.bincount(d, minlength=V)
        self.outdeg = np.bincount(s, minlength=V)

    def ext(self, v):
        return v if self.ids is None else self.ids[v]

    def create(self, monkeypatch, knobs):
        """the graph under CUGRAPH_B200_<knob> (read when the handle is created) with the build trace on"""
        from tests.gpu_util import make_graph
        for k in sr.KNOBS:
            monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)
        for k, v in knobs.items():
            monkeypatch.setenv("CUGRAPH_B200_" + k, str(v))
        monkeypatch.setenv("CUGRAPH_B200_BUILD_TRACE", "1")
        try:
            vdt = np.int32 if self.ids is None else np.int64
            if self.orientation == "csr-input":
                order = np.lexsort((self.d, self.s))
                offs = np.concatenate([[0], np.cumsum(self.outdeg)]).astype(np.int32)
                w = None if self.w is None else self.w[order]
                return make_graph(offs, self.d[order], w, input_array_format="CSR", renumber=False, weight_dtype=self.T)
            return make_graph(self.ext(self.s), self.ext(self.d), self.w, store_transposed=self.orientation == "csc",
                              symmetric=self.orientation == "symmetric", vertex_dtype=vdt, weight_dtype=self.T,
                              vertices=self.ext(np.arange(self.V)))
        finally:
            for k in list(knobs) + ["BUILD_TRACE"]:
                monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)

    def dense(self, verts, vals):
        """a (vertices, values) result by internal id"""
        v = verts.cpu().numpy()
        x = vals.cpu().numpy().astype(np.float64)
        pos = v if self.ids is None else np.argsort(self.ids)[np.searchsorted(np.sort(self.ids), v)]
        assert v.size == self.V and np.array_equal(np.sort(pos), np.arange(self.V))
        out = np.zeros(self.V)
        out[pos] = x
        return out

    def views(self, which):
        """(in-degrees, entries) of the views a driver sweeps, in the order their layouts are built: "pull" (rows =
        destinations) and, for HITS, "out" (rows = sources), which is the same view on a symmetric graph"""
        deg = {"pull": self.indeg, "out": self.outdeg}
        if self.orientation == "symmetric":
            which = which[:1]
        return [(deg[v], self.s.size) for v in which]


def rmat(scale, seed, T=np.float32, weighted=True, orientation="csc", extra_isolated=7, scattered_ids=False):
    """directed RMAT (symmetrised for "symmetric") with `extra_isolated` ids past the generated ones, weights in [1/2, 1]"""
    from oracle.rmat import rmat_edgelist
    scale = scale_of(scale)
    s, d = rmat_edgelist(scale, 16 << scale, seed=seed)
    s, d = np.asarray(s, np.int64), np.asarray(d, np.int64)
    V = (1 << scale) + extra_isolated
    w = np.random.default_rng(seed).uniform(0.5, 1.0, s.size) if weighted else None
    if orientation == "symmetric":
        s, d = np.concatenate([s, d]), np.concatenate([d, s])
        w = None if w is None else np.concatenate([w, w])
    ids = None
    if scattered_ids:
        ids = np.random.default_rng(seed + 1).choice(np.arange(10**12, 10**12 + 10**8), V, replace=False).astype(np.int64)
    return Graph(s, d, V, T, None if w is None else w.astype(T), orientation, ids,
                 f"RMAT-{scale} {np.dtype(T).name}{'w' if weighted else ''} {orientation}{' int64-ids' if ids is not None else ''}")


# ---------------------------------------------------------------------------------------------------------------------
# layouts
# ---------------------------------------------------------------------------------------------------------------------
_HEAD = re.compile(r"^\[sweep\] B=", re.M)


def check_layouts(err, graph, knobs, which, label):
    """the piece streams built while `err` was written are those that `knobs` give the views `which` of the graph"""
    es = np.dtype(graph.T).itemsize
    want = [w for w in (sr.expected_layout(deg, nnz, knobs, es, l2_bytes())
                        for deg, nnz in graph.views(which)) if w is not None]
    starts = [m.start() for m in _HEAD.finditer(err)]
    assert len(starts) == len(want), (f"{label}: {len(want)} piece stream(s) expected for the views {which}, "
                                      f"{len(starts)} built:\n{err}")
    if not want:
        sr.check_trace(err, None, label)
    for k, w in enumerate(want):
        sr.check_trace(err[starts[k]:starts[k + 1] if k + 1 < len(starts) else len(err)], w, f"{label} (view {k})")


# ---------------------------------------------------------------------------------------------------------------------
# comparison
# ---------------------------------------------------------------------------------------------------------------------
def compare(got, ref, rtol, label, key):
    """|got - ref| <= rtol |ref| everywhere, exactly 0 where ref is; records and returns the worst ratio"""
    zero = ref == 0.0
    bad_zero = np.flatnonzero(zero & (got != 0.0))
    assert bad_zero.size == 0, (f"{label}: {bad_zero.size} vertices must be exactly 0, e.g. vertex {int(bad_zero[0])} "
                                f"= {got[bad_zero[0]]!r}")
    ratio = np.zeros(ref.size)
    ratio[~zero] = np.abs(got[~zero] - ref[~zero]) / (rtol * np.abs(ref[~zero]))
    worst = float(np.nanmax(np.where(np.isnan(ratio), np.inf, ratio))) if ratio.size else 0.0
    i = int(np.argmax(np.where(np.isnan(ratio), np.inf, ratio))) if ratio.size else 0
    msg = (f"{label}: worst |got - ref| / (rtol |ref|) = {worst:.3g} at vertex {i} (got {got[i]!r}, expected {ref[i]!r}, "
           f"rtol {rtol:.3g})")
    print(msg)
    assert worst <= 1.0, msg
    WORST[key] = max(WORST[key], worst)
    return worst


def check_count(k, k_ref, diffs, thr, tol_diff, T, label):
    """the driver's iteration count against the reference's convergence step (diffs[j]: the reference's difference after
    step j + 1); one step apart only where the reference's difference at the earlier step is within tol_diff of thr"""
    if k == k_ref:
        return
    j = min(k, k_ref) - 1
    near = abs(diffs[j] - thr) <= tol_diff[j] + 2.0 * unit(T) * thr
    assert abs(k - k_ref) == 1 and near, (f"{label}: the driver stopped after {k} steps, the reference after {k_ref}; "
                                          f"reference difference at step {j + 1}: {diffs[j]!r}, threshold {thr!r}, "
                                          f"bound {tol_diff[j]:.3g}")


def run_until(step, x0, k, thr, limit):
    """run the reference `step` from x0 for k steps; also run on to find where the reference itself converges (its
    difference below thr), up to k + 1 and at most `limit` steps.  Returns (states[0..k], diffs, k_ref)"""
    xs, diffs, k_ref = [x0], [], None
    x = x0
    n = 0
    while n < max(k, 1) or (k_ref is None and n < min(k + 1, limit)):
        x, diff = step(x)
        xs.append(x)
        diffs.append(diff)
        n += 1
        if k_ref is None and diff < thr:
            k_ref = n
    return xs, diffs, k_ref if k_ref is not None else n + 1


# ---------------------------------------------------------------------------------------------------------------------
# the C entry points
# ---------------------------------------------------------------------------------------------------------------------
def _view(t):
    from cugraph_b200.pylibcugraph.utils import View
    return View(t)


def _dev(a, dtype):
    import torch
    return torch.as_tensor(np.ascontiguousarray(a, dtype=dtype)).cuda()


def centrality_call(name, h, g, *args):
    """cugraph_<name>(handle, graph, *args, ...): (vertices, values, iterations)"""
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import copy_to_torch
    L = _capi.lib()
    res, err = C.c_void_p(), C.c_void_p()
    h.order_after_caller()
    code = getattr(L, "cugraph_" + name)(h.ptr, g.ptr, *args, C.byref(res), C.byref(err))
    if res.value and code != 0:
        L.cugraph_centrality_result_free(res)
    _capi.check(code, err, "cugraph_" + name)
    verts = copy_to_torch(h, L.cugraph_centrality_result_get_vertices(res))
    vals = copy_to_torch(h, L.cugraph_centrality_result_get_values(res))
    it = int(L.cugraph_centrality_result_get_num_iterations(res))
    L.cugraph_centrality_result_free(res)
    return verts, vals, it


def hits_call(h, g, epsilon, max_iterations, guess=None, normalize=True):
    """(vertices, hubs, authorities, hub_score_differences, number_of_iterations)"""
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.utils import copy_to_torch
    L = _capi.lib()
    gv, gx = _view(guess[0] if guess else None), _view(guess[1] if guess else None)
    res, err = C.c_void_p(), C.c_void_p()
    h.order_after_caller()
    code = L.cugraph_hits(h.ptr, g.ptr, float(epsilon), int(max_iterations), gv.ptr, gx.ptr, int(normalize), 0,
                          C.byref(res), C.byref(err))
    gv.free()
    gx.free()
    _capi.check(code, err, "cugraph_hits")
    out = (copy_to_torch(h, L.cugraph_hits_result_get_vertices(res)), copy_to_torch(h, L.cugraph_hits_result_get_hubs(res)),
           copy_to_torch(h, L.cugraph_hits_result_get_authorities(res)),
           float(L.cugraph_hits_result_get_hub_score_differences(res)), int(L.cugraph_hits_result_get_number_of_iterations(res)))
    L.cugraph_hits_result_free(res)
    return out


def pagerank_call(h, g, graph, alpha, epsilon, max_iterations, pers=None, guess=None, out_w=None, expensive=False,
                  allow_nonconvergence=True):
    """cugraph_[personalized_]pagerank[_allow_nonconvergence]; pers / guess / out_w are (internal ids, values in T)"""
    vt = np.int32 if graph.ids is None else np.int64
    keep = []

    def pair(p):
        if p is None:
            return None, None
        v, x = _view(_dev(graph.ext(np.asarray(p[0])), vt)), _view(_dev(p[1], graph.T))
        keep.extend((v, x))
        return v.ptr, x.ptr
    args = [*pair(out_w), *pair(guess)]
    name = "personalized_pagerank" if pers is not None else "pagerank"
    if pers is not None:
        args += [*pair(pers)]
    args += [float(alpha), float(epsilon), int(max_iterations), int(expensive)]
    try:
        return centrality_call(name + ("_allow_nonconvergence" if allow_nonconvergence else ""), h, g, *args)
    finally:
        for v in keep:
            v.free()


# ---------------------------------------------------------------------------------------------------------------------
# Katz
# ---------------------------------------------------------------------------------------------------------------------
def katz_alpha(graph, share=0.5):
    """share / (largest in-degree * largest weight): alpha ||A||_inf <= share"""
    wmax = 1.0 if graph.w is None else float(graph.w.max())
    return share / (int(graph.indeg.max()) * wmax)


def check_katz(h, g, graph, alpha, beta, epsilon, betas=False, key=None, max_iterations=1000):
    """cugraph_katz_centrality on the graph, checked by verify_katz"""
    bv = _view(_dev(np.full(graph.V, 7.0), graph.T) if betas else None)       # the C API ignores betas
    verts, vals, k = centrality_call("katz_centrality", h, g, bv.ptr, float(alpha), float(beta), float(epsilon),
                                     int(max_iterations), 0)
    bv.free()
    return verify_katz(graph, graph.dense(verts, vals), k, alpha, beta, epsilon, key=key, max_iterations=max_iterations,
                       tag=" betas" if betas else "")


def verify_katz(graph, got, k, alpha, beta, epsilon, extra=0.0, key=None, max_iterations=1000, tag=""):
    """Katz from x = 0, x <- alpha A x + beta until sum |x - x_prev| < epsilon, then x / ||x||_2: `got` (by internal id)
    after the k steps the driver reports; `extra` is the relative rounding a sweep adds past one GPU's"""
    T, V, A = graph.T, graph.V, graph.A
    label = f"Katz {graph.label} alpha={alpha:.4g} beta={beta} epsilon={epsilon}{tag}"
    thr = float(T(epsilon))

    def step(x):
        new = alpha * (A @ x) + beta
        return new, float(np.abs(new - x).sum())
    xs, diffs, k_ref = run_until(step, np.zeros(V), k, thr, max_iterations)
    u = unit(T)
    rho = alpha * float(abs(A).sum(axis=1).max())
    assert rho < 1.0, rho
    delta = sweep_delta(T, int(graph.indeg.max())) + extra
    err = [delta * min(j, 1.0 / (1.0 - rho)) for j in range(len(xs))]
    l1 = [float(x.sum()) for x in xs]
    tol_diff = [SECOND_ORDER * (err[j + 1] * l1[j + 1] + err[j] * l1[j] + V * E * (l1[j + 1] + l1[j]))
                for j in range(len(diffs))]
    check_count(k, k_ref, diffs, thr, tol_diff, T, label)
    x = xs[k]
    ref = x / math.sqrt(float((x * x).sum()))
    rtol = SECOND_ORDER * (2.0 * err[k] + V * E + u + 2.0 * E)
    return compare(got, ref, rtol, f"{label}, {k} steps", key or f"katz {np.dtype(T).name}")


# ---------------------------------------------------------------------------------------------------------------------
# eigenvector centrality
# ---------------------------------------------------------------------------------------------------------------------
def check_eigenvector(h, g, graph, epsilon, key=None, max_iterations=1000):
    """cugraph_eigenvector_centrality on the graph, checked by verify_eigenvector"""
    verts, vals, k = centrality_call("eigenvector_centrality", h, g, float(epsilon), int(max_iterations), 0)
    return verify_eigenvector(graph, graph.dense(verts, vals), k, epsilon, key=key, max_iterations=max_iterations)


def verify_eigenvector(graph, got, k, epsilon, extra=0.0, key=None, max_iterations=1000, tag=""):
    """x <- (A x + x) / ||A x + x||_2 from x = 1/V until sum |x - x_prev| < V epsilon: `got` (by internal id) after the
    k steps the driver reports; `extra` is the relative rounding a sweep adds past one GPU's"""
    T, V, A = graph.T, graph.V, graph.A
    label = f"eigenvector {graph.label} epsilon={epsilon}{tag}"
    thr = float(T(V) * T(epsilon))

    def step(x):
        y = A @ x + x
        y = y / math.sqrt(float((y * y).sum()))
        return y, float(np.abs(y - x).sum())
    xs, diffs, k_ref = run_until(step, np.full(V, 1.0 / V), k, thr, max_iterations)
    u = unit(T)
    theta = V * E + u + 2.0 * E
    D = [2.0 * j * (sweep_delta(T, int(graph.indeg.max())) + extra + 2.0 * u + 2.0 * E) for j in range(len(xs))]
    rt = [SECOND_ORDER * (math.expm1(Dj) + theta) for Dj in D]
    l1 = [float(x.sum()) for x in xs]
    tol_diff = [rt[j + 1] * l1[j + 1] + rt[j] * l1[j] + V * E * (l1[j + 1] + l1[j]) for j in range(len(diffs))]
    check_count(k, k_ref, diffs, thr, tol_diff, T, label)
    return compare(got, xs[k], rt[k], f"{label}, {k} steps", key or f"eigenvector {np.dtype(T).name}")


# ---------------------------------------------------------------------------------------------------------------------
# HITS
# ---------------------------------------------------------------------------------------------------------------------
def check_hits(h, g, graph, epsilon, guess=None, normalize=True, key=None, max_iterations=1000):
    """cugraph_hits on the graph, checked by verify_hits"""
    gd = None
    if guess is not None:
        vt = np.int32 if graph.ids is None else np.int64
        gd = (_dev(graph.ext(np.asarray(guess[0])), vt), _dev(guess[1], graph.T))
    verts, hubs, auth, hdiff, k = hits_call(h, g, epsilon, max_iterations, gd, normalize)
    return verify_hits(graph, graph.dense(verts, hubs), graph.dense(verts, auth), hdiff, k, epsilon, guess, normalize,
                       key=key, max_iterations=max_iterations)


def verify_hits(graph, hubs, auth, hdiff, k, epsilon, guess=None, normalize=True, extra=(0.0, 0.0), key=None,
                max_iterations=1000, tag=""):
    """authorities = N hubs, hubs = N^T authorities (N: the unweighted multigraph), both divided by their maximum, until
    sum |hubs - hubs_prev| < V epsilon; divided by their sums with `normalize`.  guess = (internal ids, values): the
    initial hubs, 0 for the vertices it leaves out, divided by their sum.  hubs, auth (by internal id), hdiff
    (hub_score_differences) and k as the driver reports them; extra = (pull, transposed): the relative rounding each of the
    two sweeps adds past one GPU's"""
    T, V, N, Nt = graph.T, graph.V, graph.N, graph.Nt
    label = (f"HITS {graph.label} epsilon={epsilon} normalize={normalize}"
             f"{f' guess on {len(guess[0])} vertices' if guess is not None else ''}{tag}")
    thr = float(T(V) * T(epsilon))
    if guess is None:
        h0 = np.full(V, 1.0 / V)
    else:
        h0 = np.zeros(V)
        h0[np.asarray(guess[0])] = np.asarray(guess[1], T).astype(np.float64)
        h0 /= h0.sum()
    auths = {}

    def step(hv):
        a = N @ hv
        c = Nt @ a
        c, a = c / c.max(), a / a.max()
        auths[id(c)] = a
        return c, float(np.abs(c - hv).sum())
    xs, diffs, k_ref = run_until(step, h0, k, thr, max_iterations)
    u = unit(T)
    d_in = sweep_delta(T, int(graph.indeg.max())) + extra[0]
    d_out = sweep_delta(T, int(graph.outdeg.max())) + extra[1]
    D0 = 2.0 * (u + 2.0 * E) if guess is not None else 0.0
    Dh = [D0 + 2.0 * j * (d_in + d_out + u + 2.0 * E) for j in range(len(xs))]
    rt = [SECOND_ORDER * math.expm1(Dj) for Dj in Dh]
    l1 = [float(x.sum()) for x in xs]
    tol_diff = [rt[j + 1] * l1[j + 1] + rt[j] * l1[j] + V * E * (l1[j + 1] + l1[j]) for j in range(len(diffs))]
    check_count(k, k_ref, diffs, thr, tol_diff, T, label)
    j = k - 1
    assert abs(hdiff - diffs[j]) <= tol_diff[j] + 2.0 * u * diffs[j], \
        f"{label}: hub_score_differences {hdiff!r}, reference {diffs[j]!r}, bound {tol_diff[j]:.3g}"
    ref_h, ref_a = xs[k], auths[id(xs[k])]
    rt_h = math.expm1(Dh[k])
    rt_a = math.expm1(Dh[k - 1] + 2.0 * (d_in + u + 2.0 * E))
    if normalize:
        ref_h, ref_a = ref_h / ref_h.sum(), ref_a / ref_a.sum()
        rt_h, rt_a = rt_h + V * E + u + 2.0 * E, rt_a + V * E + u + 2.0 * E
    key = key or f"hits {np.dtype(T).name}"
    w1 = compare(hubs, ref_h, SECOND_ORDER * rt_h, f"{label}, hubs after {k} steps", key)
    w2 = compare(auth, ref_a, SECOND_ORDER * rt_a, f"{label}, authorities after {k} steps", key)
    return max(w1, w2)


# ---------------------------------------------------------------------------------------------------------------------
# PageRank
# ---------------------------------------------------------------------------------------------------------------------
def check_pagerank(h, g, graph, steps=30, alpha=0.85, pers=None, guess=None, out_w=None, key=None):
    """`steps` steps of cugraph_[personalized_]pagerank at epsilon = 0, checked by verify_pagerank"""
    verts, vals, k = pagerank_call(h, g, graph, alpha, 0.0, steps, pers, guess, out_w)
    return verify_pagerank(graph, graph.dense(verts, vals), k, steps, alpha, pers, guess, out_w, key=key)


def verify_pagerank(graph, got, k, steps=30, alpha=0.85, pers=None, guess=None, out_w=None, extra=0.0, key=None, tag=""):
    """`got` (by internal id) after `steps` steps at epsilon = 0 (k: the count the driver reports) against oracle.pagerank;
    pers / guess / out_w: (internal ids, values in T); `extra` is the relative rounding a sweep adds past one GPU's"""
    import oracle
    T, V = graph.T, graph.V
    parts = [n for n, p in (("personalized", pers), ("initial guess", guess), ("out-weights", out_w)) if p is not None]
    label = f"PageRank {graph.label}{' ' + ', '.join(parts) if parts else ''}{tag}"
    assert k == steps, f"{label}: {k} steps at epsilon 0, expected {steps}"

    def dense(p):
        x = np.zeros(V)
        x[np.asarray(p[0])] = np.asarray(p[1], T).astype(np.float64)
        return x
    w = None if graph.w is None else graph.w.astype(np.float64)
    ref, _, _ = oracle.pagerank(graph.s, graph.d, V, w, alpha=alpha, epsilon=0.0, max_iterations=steps,
                                personalization=None if pers is None else (np.asarray(pers[0], np.int32),
                                                                           np.asarray(pers[1], T).astype(np.float64)),
                                initial_guess=None if guess is None else dense(guess),
                                precomputed_out_w=None if out_w is None else dense(out_w))
    u = unit(T)
    n_pers = 0 if pers is None else len(pers[0])
    per_step = (sweep_delta(T, int(graph.indeg.max())) + extra + 3.0 * u + (int(graph.outdeg.max()) + V + n_pers) * E
                + 8.0 * E)
    rtol = SECOND_ORDER * (u + steps * per_step)
    return compare(got, ref, rtol, f"{label}, {steps} steps",
                   key or f"{'personalized ' if pers is not None else ''}pagerank {np.dtype(T).name}")


def personalizations(graph, seed=0):
    """tests/mg_pagerank_ref.cases: one hub, a sink, a vertex without in-edges, an isolated id, a share with zeros among
    the values — as (internal ids, values)"""
    from tests.mg_pagerank_ref import cases
    V = graph.V
    share = np.random.default_rng(seed).choice(V, size=max(V // 8, 2), replace=False)   # the draw of cases(): its zeros too
    out = {}
    for name, pv in cases(graph.s, graph.d, V, seed).items():
        ids = share if name == "share_with_zeros" else np.flatnonzero(pv)
        out[name] = (ids.astype(np.int64), pv[ids].astype(graph.T))
    assert (out["share_with_zeros"][1] == 0).sum() > 0
    return out


# ---------------------------------------------------------------------------------------------------------------------
# cases: a graph under a layout, each algorithm's calls on it, and the layouts they built
# ---------------------------------------------------------------------------------------------------------------------
TYPES = {"f32w": (np.float32, True), "f64w": (np.float64, True), "f32": (np.float32, False)}
_GRAPHS = {}


def graph_of(etype, scale, orientation="csc", scattered_ids=False):
    """directed RMAT at `scale` (the emulation's cap applied), cached per module run"""
    key = (etype, scale_of(scale), orientation, scattered_ids)
    if key not in _GRAPHS:
        T, weighted = TYPES[etype]
        _GRAPHS[key] = rmat(scale, 900 + scale + 7 * len(_GRAPHS), T, weighted, orientation, scattered_ids=scattered_ids)
    return _GRAPHS[key]


def epsilons(graph):
    """Katz: epsilon of 1e-6 (float32) / 1e-14 (float64) per vertex; eigenvector and HITS: thresholds V epsilon a decade or
    more above the difference at which rounding leaves the iteration.  RMAT's large spectral gap makes all three converge
    fast: 4-7 steps in float32, 8-11 in float64"""
    f32 = graph.T == np.float32
    return {"katz": graph.V * (1e-6 if f32 else 1e-14), "eigenvector": 1e-8 if f32 else 1e-15, "hits": 1e-8 if f32 else 1e-15}


def run_case(algorithm, monkeypatch, capfd, graph, layout):
    """the checks of one algorithm on `graph` built under KNOBS[layout]; returns the worst observed / bound"""
    knobs = KNOBS[layout]
    capfd.readouterr()
    h, g = graph.create(monkeypatch, knobs)
    eps = epsilons(graph)
    t = np.dtype(graph.T).name
    worst = 0.0
    views = ["pull"]
    if algorithm == "katz":
        a = katz_alpha(graph)
        worst = max(check_katz(h, g, graph, a, 1.0, eps["katz"]),
                    check_katz(h, g, graph, a, 0.25, 0.25 * eps["katz"], betas=True),
                    check_katz(h, g, graph, katz_alpha(graph, 0.9), 1.0, eps["katz"], key=f"katz {t} near the limit"))
    elif algorithm == "eigenvector":
        worst = check_eigenvector(h, g, graph, eps["eigenvector"])
    elif algorithm == "hits":
        views = ["pull", "out"]
        rng = np.random.default_rng(3)
        part = np.sort(rng.choice(graph.V, graph.V // 3, replace=False))
        guess = (part, rng.uniform(0.1, 1.0, part.size).astype(graph.T))
        worst = max(check_hits(h, g, graph, eps["hits"]),
                    check_hits(h, g, graph, eps["hits"], guess=guess, normalize=False))
    elif algorithm == "personalized":
        steps = 10 if emulated() else 30        # the emulation runs a launch's threads one after the other
        for p in personalizations(graph).values():
            worst = max(worst, check_pagerank(h, g, graph, steps=steps, pers=p))
        rng = np.random.default_rng(4)
        guess = (np.arange(graph.V), rng.uniform(0.0, 2.0 / graph.V, graph.V).astype(graph.T))
        ow = np.bincount(graph.s, weights=None if graph.w is None else graph.w.astype(np.float64), minlength=graph.V)
        out_w = (np.arange(graph.V), (2.0 * ow).astype(graph.T))
        worst = max(worst, check_pagerank(h, g, graph, steps=steps, pers=personalizations(graph)["share_with_zeros"],
                                          guess=guess, out_w=out_w))
    else:
        raise ValueError(algorithm)
    check_layouts(capfd.readouterr().err, graph, knobs, views, f"{algorithm} {graph.label} {layout}")
    return worst


def run_many_calls(monkeypatch, capfd, graph, layout):
    """one graph through PageRank, Katz, HITS, eigenvector, personalized PageRank, PageRank with precomputed out-weights
    (twice the true sums) and plain PageRank again, each against its reference"""
    knobs = KNOBS[layout]
    capfd.readouterr()
    h, g = graph.create(monkeypatch, knobs)
    eps = epsilons(graph)
    check_pagerank(h, g, graph)
    check_katz(h, g, graph, katz_alpha(graph), 1.0, eps["katz"])
    check_hits(h, g, graph, eps["hits"])
    check_eigenvector(h, g, graph, eps["eigenvector"])
    check_pagerank(h, g, graph, pers=personalizations(graph)["share_with_zeros"])
    ow = np.bincount(graph.s, weights=None if graph.w is None else graph.w.astype(np.float64), minlength=graph.V)
    check_pagerank(h, g, graph, out_w=(np.arange(graph.V), (2.0 * ow).astype(graph.T)))
    check_pagerank(h, g, graph)          # the cached out-weight sums, not the precomputed ones
    check_layouts(capfd.readouterr().err, graph, knobs, ["pull", "out"], f"many calls {graph.label} {layout}")
