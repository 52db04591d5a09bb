"""One pull sweep, checked row by row against an fp64 reference: the harness of tests/test_sweep_rows_gpu.py (the H100) and
tests/test_sweep_rows_cpu.py (the emulation build of the library, tests/emu_py.py).

A block (cugraph_b200_block_create: binned rows with row_vertex, multi-edges kept) is built from an edge list under a set of
sweep knobs, then swept three times into the same y, each time with a fresh x and another alpha.  After every sweep each row
must satisfy

    |y - y*| <= 2 * (S * (4 u_T + d 2^-52) + u_T |y*|),   y* = alpha A x,  S = |alpha| |A| |x|,  d = entries of the row,

with A the fp64 matrix of the edge list (duplicates summed) and u_T the unit roundoff of the element type (2^-24 for fp32,
2^-53 for fp64).  The bound follows the kernels' arithmetic: every product x_c w_c is rounded once in T (u_T |x_c w_c|); a
lane adds at most 8 of them in T before converting to fp64 (slot_sum: a tree of depth 3; pair_sum and the tail's batches
less), which costs at most 3 u_T per term; everything after that is fp64 — slots, pieces, REDs into the accumulator, the tail's
batches, and the reference's own sum — at most d additions of terms bounded by S, so d 2^-53 S for each of the two sums;
the final rounding to T adds u_T |y|.  Summed: S (4 u_T + 2 d 2^-53) + u_T |y*|, doubled for second-order terms and the
plain sweep's order of operations.

The inputs make a wrong row loud: |x| in [1/2, 1] with random signs and weights in [1/2, 1] put S within a factor of 2 of the
number of entries, so one dropped, doubled or misweighted entry (|x_c w_c| >= 1/4) exceeds the bound by orders of magnitude
for any row below ~10^5 entries.  x is NaN on every column below the span that no edge reads and zero from the span on — what
the block sweep's contract allows — so a stray gather (a wrong local id, block or padding column) makes y non-finite.  Rows
without edges must read exactly 0 after the first sweep into a fresh y; they are then overwritten with a sentinel that the
later sweeps of the piece stream into the same y must leave in place (the plain sweep writes 0 to them again).

CUGRAPH_B200_BUILD_TRACE=1 makes the layout builder print its shape; every case asserts that the layout it meant to run
(stream rows, tail rows, bands, tail runs / tiles / work units, or the plain sweep) is what was built."""
import ctypes as C
import re

import numpy as np

INT32, FLOAT32, FLOAT64 = 2, 8, 9
SLICE_BYTES = 192 * 1024         # kHotSliceBytes
ZERO_PAD = 64                    # kHotZeroPad
BAND_ALIGN = 512                 # kBandRowAlign
THRESHOLDS = (32, 16, 8, 4, 2, 1)
TAIL_UNIT_ENTRIES = 24           # kTailUnitEntries
DEFAULT_MIN_EDGES = 1 << 22      # tuning_t::sweep_min_edges
DEFAULT_OFFS64_EDGES = 1 << 31
TAIL_MIN_EDGES = 1 << 24         # kSweepTailMinEdges
TAIL_DEFAULT = 16                # kSweepTailDegree
ALPHAS = (0.85, 1.0, -0.5)
SENTINEL = 1234.5
KNOBS = ("SWEEP_MIN_EDGES", "SWEEP_BANDS", "SWEEP_TAIL_DEGREE", "SWEEP_BANK_ORDER", "OFFS64_MIN_EDGES")


def W_of(es):
    return SLICE_BYTES // es - ZERO_PAD


def unit_tiles(d):
    return 1 if d >= TAIL_UNIT_ENTRIES else TAIL_UNIT_ENTRIES // d


def threshold(bound):
    """the bin bound the builder rounds a tail bound down to (sweep_stream_bin)"""
    return next(t for t in THRESHOLDS if t <= bound)


def expected_layout(deg, nnz, knobs, es, l2_bytes):
    """what the builder must make of a block whose rows have in-degrees `deg`, or None for the plain sweep"""
    min_edges = int(knobs.get("SWEEP_MIN_EDGES", DEFAULT_MIN_EDGES))
    offs64 = nnz >= min(max(int(knobs.get("OFFS64_MIN_EDGES", DEFAULT_OFFS64_EDGES)), 0), 1 << 31)
    n_cov = int((deg >= 1).sum())
    if nnz < min_edges or offs64 or n_cov == 0:
        return None
    bound = int(knobs.get("SWEEP_TAIL_DEGREE", 0))
    if bound <= 0:
        bound = TAIL_DEFAULT if nnz >= TAIL_MIN_EDGES else 1
    thr = threshold(bound)
    n_str = int((deg >= thr).sum())
    if n_str == 0:
        return None
    most = max(1, -(-n_str // BAND_ALIGN))
    P = int(knobs.get("SWEEP_BANDS", 0))
    if P <= 0:
        P = int(np.ceil(8.0 * n_str / (0.5 * l2_bytes))) if l2_bytes else 1
    asked = min(max(P, 1), most)
    band_rows = -(-(-(-n_str // asked)) // BAND_ALIGN) * BAND_ALIGN
    runs = tiles = units = 0
    for d in range(1, thr):
        n = int((deg == d).sum())
        if n:
            t = -(-n // 32)
            runs, tiles, units = runs + 1, tiles + t, units + -(-t // unit_tiles(d))
    return {"W": W_of(es), "B": -(-deg.size // W_of(es)), "rows": n_str, "tail": n_cov - n_str, "thr": thr,
            "bands": -(-n_str // band_rows), "band_rows": band_rows, "runs": runs, "tiles": tiles, "units": units}


_HEAD = re.compile(r"\[sweep\] B=(\d+) W=(\d+) rows=(\d+) \(tail (\d+) rows, \d+ edges\) .* bands=(\d+) of (\d+) rows")
_TAIL = re.compile(r"\[sweep\] tail: (\d+) runs, (\d+) tiles, (\d+) units")


def check_trace(err, want, label):
    if want is None:
        assert "[sweep]" not in err, f"{label}: the plain sweep was expected, the builder made a piece stream:\n{err}"
        return
    m = _HEAD.search(err)
    assert m, f"{label}: no piece-stream trace line in:\n{err}"
    got = dict(zip(("B", "W", "rows", "tail", "bands", "band_rows"), map(int, m.groups())))
    for k, v in got.items():
        assert v == want[k], f"{label}: {k}={v}, expected {want[k]} ({got} vs {want})"
    t = _TAIL.search(err)
    if want["tail"] == 0:
        assert t is None, f"{label}: a tail layout without tail rows"
        return
    assert t, f"{label}: no tail trace line in:\n{err}"
    got = dict(zip(("runs", "tiles", "units"), map(int, t.groups())))
    for k, v in got.items():
        assert v == want[k], f"{label}: tail {k}={v}, expected {want[k]}"


def reference(rows, cols, w, n_span, n_cols):
    """fp64 CSR of the edge list over [0, n_span) rows (duplicates summed), and each row's entry count"""
    import scipy.sparse as sp
    vals = np.ones(rows.size) if w is None else w.astype(np.float64)
    A = sp.csr_matrix((vals, (rows.astype(np.int64), cols.astype(np.int64))), shape=(n_span, n_span))
    A.sum_duplicates()
    return A, np.bincount(rows, minlength=n_span)


def diagnose(y, ys, tol, ratio, deg, layout, rows, cols, w, x, alpha, label, k):
    r = int(np.nanargmax(np.where(np.isnan(ratio), np.inf, ratio)))
    d = int(deg[r])
    if d == 0:
        kind = "empty row"
    elif layout is None:
        kind = "plain sweep row"
    elif d >= layout["thr"]:
        kind = "stream row"
    else:
        kind = f"tail row (run degree {d})"
    diff = float(y[r]) - ys[r]
    m = rows == r
    c, ww = cols[m], (np.ones(int(m.sum())) if w is None else w[m].astype(np.float64))
    hit = [int(cc) for cc, v in zip(c, alpha * x[c].astype(np.float64) * ww)
           if abs(diff - v) <= tol[r] or abs(diff + v) <= tol[r]]
    entry = f"; the difference is +-x_c*w_c of column(s) {sorted(set(hit))[:8]}" if hit else ""
    return (f"{label}, sweep {k} (alpha {alpha}): {int(np.sum(~(np.abs(y - ys) <= tol)))} rows out of bound; worst row {r} "
            f"({kind}, {d} entries): got {float(y[r])!r}, expected {ys[r]!r}, tol {tol[r]:.3g}{entry}")


def run_block(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, label, seed=0):
    """build the block under `knobs`, sweep it three times, check every row after every sweep; returns the largest
    |y - y*| / tol over the sweeps"""
    import torch
    for k in KNOBS:
        monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)
    for k, v in knobs.items():
        monkeypatch.setenv("CUGRAPH_B200_" + k, str(v))
    monkeypatch.setenv("CUGRAPH_B200_BUILD_TRACE", "1")      # read when the handle is created
    es = 8 if dtype == np.float64 else 4
    tt = torch.float64 if es == 8 else torch.float32
    tid = FLOAT64 if es == 8 else FLOAT32
    u = 2.0 ** -53 if es == 8 else 2.0 ** -24
    rows = np.ascontiguousarray(rows, dtype=np.int32)
    cols = np.ascontiguousarray(cols, dtype=np.int32)
    n_span = max(n_rows, n_cols)
    capfd.readouterr()
    handle = C.c_void_p(lib.cugraph_b200_create_resource_handle_on_stream(C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert handle.value
    keep, views = [], []

    def view(t, type_id):
        keep.append(t)
        v = C.c_void_p(lib.cugraph_type_erased_device_array_view_create(C.c_void_p(t.data_ptr()), t.numel(), type_id))
        views.append(v)
        return v

    blk, err = C.c_void_p(), C.c_void_p()
    try:
        vr = view(torch.from_numpy(rows).cuda(), INT32)
        vc = view(torch.from_numpy(cols).cuda(), INT32)
        vw = None if w is None else view(torch.from_numpy(np.ascontiguousarray(w, dtype=dtype)).cuda(), tid)
        code = lib.cugraph_b200_block_create(handle, n_rows, n_cols, vr, vc, vw, C.byref(blk), C.byref(err))
        assert code == 0, lib.cugraph_error_message(err)
        torch.cuda.synchronize()
        assert lib.cugraph_b200_block_span(blk) == n_span
        A, deg = reference(rows, cols, w, n_span, n_cols)
        want = expected_layout(deg, rows.size, knobs, es, l2_bytes)
        check_trace(capfd.readouterr().err, want, label)
        absA = abs(A)
        wq = None if w is None else np.asarray(w, dtype=dtype)
        x_elems = int(lib.cugraph_b200_padded_elems(n_span, es))
        read = np.zeros(n_span, bool)
        read[cols] = True
        empty = deg == 0
        rng = np.random.default_rng(seed)
        y = torch.full((n_span,), float("nan"), dtype=tt, device="cuda")   # alive until the block is freed: the block knows
        vy = view(y, tid)                                                    # "the same y" by its address
        worst = 0.0
        for k, alpha in enumerate(ALPHAS):
            xh = np.zeros(x_elems, dtype)
            xh[:n_span] = rng.uniform(0.5, 1.0, n_span) * rng.choice((-1.0, 1.0), n_span)
            xh[:n_span][~read] = np.nan
            x = torch.from_numpy(xh).cuda()
            vx = view(x, tid)
            code = lib.cugraph_b200_block_pull_sweep(handle, blk, vx, vy, alpha, C.byref(err))
            assert code == 0, lib.cugraph_error_message(err)
            torch.cuda.synchronize()
            yh = y.cpu().numpy().astype(np.float64)
            x64 = np.where(read, xh[:n_span].astype(np.float64), 0.0)
            ys = alpha * (A @ x64)
            S = abs(alpha) * (absA @ np.abs(x64))
            tol = 2.0 * (S * (4.0 * u + deg * 2.0 ** -52) + u * np.abs(ys))
            fill = SENTINEL if k > 0 and want is not None else 0.0     # the plain sweep rewrites every row
            assert np.array_equal(yh[empty], np.full(int(empty.sum()), fill)), \
                f"{label}, sweep {k}: rows without edges hold {np.unique(yh[empty])[:5]}, expected {fill}"
            ratio = np.abs(yh - ys) / np.where(tol > 0, tol, 1.0)
            ratio[empty] = 0.0
            if not np.all(ratio[~empty] <= 1.0):       # NaN fails too
                raise AssertionError(diagnose(yh, ys, tol, ratio, deg, want, rows, cols, wq, xh, alpha, label, k))
            worst = max(worst, float(ratio.max()))
            if k == 0:                                  # later sweeps into this y must leave these entries alone
                y[torch.from_numpy(np.nonzero(empty)[0]).cuda()] = SENTINEL
        return worst
    finally:
        if blk.value:
            lib.cugraph_b200_block_free(blk)
        for v in views:
            lib.cugraph_type_erased_device_array_view_free(v)
        lib.cugraph_free_resource_handle(handle)


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
def run_lengths(d):
    """the tail run lengths that put a run's end at and around tile and work-unit bounds"""
    k = unit_tiles(d)
    return (1, 31, 32, 33, 32 * k - 1, 32 * k, 32 * k + 1, 32 * k * 3 + 17)


def ladder(seed=0, n_hubs=2301, n_cols=122_741, n_rows=None):
    """rows of every in-degree 1..31 (run lengths rotated by `seed` through run_lengths), n_hubs rows of in-degree 32 to
    ~3000 (one of them with more than 2048 entries in column block 0, one with entries in every block), the columns next to
    the block bounds of both element widths, duplicate entries, and empty rows.  Column 0 is never read."""
    rng = np.random.default_rng(1000 + seed)
    n_rows = n_cols if n_rows is None else n_rows
    degs = [d for d in range(1, 32) for _ in range(run_lengths(d)[(d + seed) % 8])]
    hub = np.minimum(32 + (rng.pareto(1.2, n_hubs) * 20).astype(np.int64), 3000)
    hub[0], hub[1] = 2600, 3000
    degs = np.concatenate([hub, np.array(degs, np.int64)])
    assert degs.size < n_rows
    row_ids = rng.permutation(n_rows)[:degs.size]                  # row slots: arbitrary, the rest stay empty
    rows = np.repeat(row_ids, degs)
    cols = rng.integers(1, n_cols, rows.size)
    start = np.concatenate([[0], np.cumsum(degs)])
    W4, W8 = W_of(4), W_of(8)
    cols[start[0]:start[1]] = rng.integers(1, W8, 2600)             # > 2048 entries in block 0 of either width
    special = sorted({W - 1 for W in (W4, W8)} | {W for W in (W4, W8)} | {W + 1 for W in (W4, W8)} |
                     {2 * W - 1 for W in (W4, W8)} | {2 * W for W in (W4, W8)} | {n_cols - 1} |
                     {b * W8 + 7 for b in range(-(-n_cols // W8))})
    cols[start[1]:start[1] + len(special)] = special                # this row touches every block
    for i in range(2, 40):                                          # duplicate (row, col) pairs, hubs and tail rows
        a = start[i]
        cols[a + 1] = cols[a]
    for d_row in np.nonzero((degs >= 2) & (degs < 32))[0][::97]:
        a = start[d_row]
        cols[a + 1] = cols[a]
    return rows.astype(np.int32), cols.astype(np.int32), n_rows, n_cols


def stream_rows(rows, n_span, thr):
    return int((np.bincount(rows, minlength=n_span) >= thr).sum())


def random_block(n_rows, n_cols, n_hubs, n_low, seed):
    """a rectangular block: n_hubs rows of in-degree 32..~500 and n_low rows of in-degree 1..31"""
    rng = np.random.default_rng(seed)
    degs = np.concatenate([np.minimum(32 + (rng.pareto(1.5, n_hubs) * 30).astype(np.int64), 500),
                           rng.integers(1, 32, n_low)])
    row_ids = rng.permutation(n_rows)[:degs.size]
    rows = np.repeat(row_ids, degs)
    cols = rng.integers(0, n_cols, rows.size)
    return rows.astype(np.int32), cols.astype(np.int32)


def weights(n, dtype, seed):
    return np.random.default_rng(seed).uniform(0.5, 1.0, n).astype(dtype)
