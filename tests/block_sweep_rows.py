"""The block sweep in both orientations (cugraph_b200_block_sweep), checked row by row against an fp64 reference with the
bound, inputs and layout traces of tests/sweep_rows.py: the harness of tests/test_block_sweep_rows_cpu.py (the emulation build
of the library) and tests/test_block_sweep_rows_gpu.py (the H100).

The transposed sweep y[col] = alpha * sum over the edges (row, col) of x[row] * w is the pull sweep of the block's
column-major copy, so its reference is sweep_rows.reference(cols, rows, ...) and its layout is what sweep_rows.expected_layout
makes of the column in-degrees.  x is indexed by row slot: NaN where no edge reads, zero from the span on.  Every case sweeps
three times (alphas 0.85 / 1 / -0.5) into one y per orientation: empty slots read 0 after the first sweep, then hold a
sentinel that the piece stream's later sweeps into the same y must leave alone."""
import ctypes as C

import numpy as np

from tests import sweep_rows as sr


class Case:
    """one block under a set of sweep knobs, with a y per orientation"""

    def __init__(self, lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, label):
        import torch
        self.torch, self.lib, self.capfd, self.label = torch, lib, capfd, label
        for k in sr.KNOBS:
            monkeypatch.delenv("CUGRAPH_B200_" + k, raising=False)
        for k, v in knobs.items():
            monkeypatch.setenv("CUGRAPH_B200_" + k, str(v))
        monkeypatch.setenv("CUGRAPH_B200_BUILD_TRACE", "1")      # read when the handle is created
        self.es = 8 if dtype == np.float64 else 4
        self.dtype = dtype
        self.tt = torch.float64 if self.es == 8 else torch.float32
        self.tid = sr.FLOAT64 if self.es == 8 else sr.FLOAT32
        self.u = 2.0 ** -53 if self.es == 8 else 2.0 ** -24
        self.rows = np.ascontiguousarray(rows, dtype=np.int32)
        self.cols = np.ascontiguousarray(cols, dtype=np.int32)
        self.w = w
        self.knobs, self.l2_bytes = knobs, l2_bytes
        self.n_span = max(n_rows, n_cols)
        capfd.readouterr()
        self.handle = C.c_void_p(lib.cugraph_b200_create_resource_handle_on_stream(
            C.c_void_p(torch.cuda.current_stream().cuda_stream)))
        assert self.handle.value
        self.keep, self.views = [], []
        self.blk, self.err = C.c_void_p(), C.c_void_p()
        vr = self.view(torch.from_numpy(self.rows).cuda(), sr.INT32)
        vc = self.view(torch.from_numpy(self.cols).cuda(), sr.INT32)
        vw = None if w is None else self.view(torch.from_numpy(np.ascontiguousarray(w, dtype=dtype)).cuda(), self.tid)
        code = lib.cugraph_b200_block_create(self.handle, n_rows, n_cols, vr, vc, vw, C.byref(self.blk), C.byref(self.err))
        assert code == 0, lib.cugraph_error_message(self.err)
        torch.cuda.synchronize()
        self.pull_trace = capfd.readouterr().err
        self.x_elems = int(lib.cugraph_b200_padded_elems(self.n_span, self.es))
        self.rng = np.random.default_rng(0)
        self.y = {}

    def view(self, t, type_id):
        self.keep.append(t)
        v = C.c_void_p(self.lib.cugraph_type_erased_device_array_view_create(C.c_void_p(t.data_ptr()), t.numel(), type_id))
        self.views.append(v)
        return v

    def free(self):
        if self.blk.value:
            self.lib.cugraph_b200_block_free(self.blk)
        for v in self.views:
            self.lib.cugraph_type_erased_device_array_view_free(v)
        self.lib.cugraph_free_resource_handle(self.handle)

    def orientation(self, transposed, use_weights):
        """(A, entries per slot, slots x reads, expected layout) of one orientation"""
        w = self.w if use_weights else None
        major, minor = (self.cols, self.rows) if transposed else (self.rows, self.cols)
        A, deg = sr.reference(major, minor, w, self.n_span, self.n_span)
        read = np.zeros(self.n_span, bool)
        read[minor] = True
        want = sr.expected_layout(deg, self.rows.size, self.knobs, self.es, self.l2_bytes)
        return A, deg, read, want

    def sweep(self, key, transposed, use_weights, alpha, entry="block_sweep"):
        """one sweep into the y named `key` (created NaN-filled on first use); returns (y as fp64, x as the element type)"""
        torch = self.torch
        if key not in self.y:
            y = torch.full((self.n_span,), float("nan"), dtype=self.tt, device="cuda")
            self.y[key] = (y, self.view(y, self.tid))
        y, vy = self.y[key]
        _, _, read, _ = self.orientation(transposed, use_weights)
        xh = np.zeros(self.x_elems, self.dtype)
        xh[:self.n_span] = self.rng.uniform(0.5, 1.0, self.n_span) * self.rng.choice((-1.0, 1.0), self.n_span)
        xh[:self.n_span][~read] = np.nan
        vx = self.view(torch.from_numpy(xh).cuda(), self.tid)
        if entry == "pull_sweep":
            code = self.lib.cugraph_b200_block_pull_sweep(self.handle, self.blk, vx, vy, alpha, C.byref(self.err))
        else:
            code = self.lib.cugraph_b200_block_sweep(self.handle, self.blk, int(transposed), int(use_weights), vx, vy, alpha,
                                                     C.byref(self.err))
        assert code == 0, self.lib.cugraph_error_message(self.err)
        torch.cuda.synchronize()
        return y.cpu().numpy().astype(np.float64), xh

    def check(self, yh, xh, transposed, use_weights, alpha, k, label):
        """the bound of tests/sweep_rows.py on every slot; empty slots 0 after sweep 0, the sentinel afterwards (piece stream)"""
        A, deg, read, want = self.orientation(transposed, use_weights)
        x64 = np.where(read, xh[:self.n_span].astype(np.float64), 0.0)
        ys = alpha * (A @ x64)
        S = abs(alpha) * (abs(A) @ np.abs(x64))
        tol = 2.0 * (S * (4.0 * self.u + deg * 2.0 ** -52) + self.u * np.abs(ys))
        empty = deg == 0
        fill = sr.SENTINEL if k > 0 and want is not None else 0.0
        assert np.array_equal(yh[empty], np.full(int(empty.sum()), fill)), \
            f"{label}, sweep {k}: slots without edges hold {np.unique(yh[empty])[:5]}, expected {fill}"
        ratio = np.abs(yh - ys) / np.where(tol > 0, tol, 1.0)
        ratio[empty] = 0.0
        if not np.all(ratio[~empty] <= 1.0):
            major, minor = (self.cols, self.rows) if transposed else (self.rows, self.cols)
            w = self.w if use_weights else None
            raise AssertionError(sr.diagnose(yh, ys, tol, ratio, deg, want, major, minor, w, xh, alpha, label, k))
        return empty

    def set_sentinel(self, key, empty):
        y, _ = self.y[key]
        y[self.torch.from_numpy(np.nonzero(empty)[0]).cuda()] = sr.SENTINEL


def run(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, label, use_weights=True,
        interleave=False, first=None):
    """three transposed sweeps into one y, checked row by row, with the transposed layout's trace checked after the first;
    interleave: a pull sweep into a second y after every transposed one, each y keeping its own covered-slots state;
    first = "wcc" / "sssp": that call builds the column-major copy before the first transposed sweep"""
    case = Case(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, label)
    try:
        if first is not None:
            _build_push_copy_first(case, first)
        case.capfd.readouterr()
        for k, alpha in enumerate(sr.ALPHAS):
            yh, xh = case.sweep("t", True, use_weights, alpha)
            if k == 0:
                sr.check_trace(case.capfd.readouterr().err, case.orientation(True, use_weights)[3], f"{label} (transposed)")
            empty = case.check(yh, xh, True, use_weights, alpha, k, f"{label} transposed")
            if k == 0:
                case.set_sentinel("t", empty)
            if interleave:
                yh, xh = case.sweep("p", False, use_weights, alpha)
                empty_p = case.check(yh, xh, False, use_weights, alpha, k, f"{label} pull")
                if k == 0:
                    case.set_sentinel("p", empty_p)
    finally:
        case.free()


def _build_push_copy_first(case, which):
    import torch
    lib = case.lib
    if which == "wcc":
        lab = torch.full((case.n_span,), np.iinfo(np.int64).max, dtype=torch.int64, device="cuda")
        cand = torch.empty(case.n_span, dtype=torch.int64, device="cuda")
        vl, vc = case.view(lab, 3), case.view(cand, 3)
        code = lib.cugraph_b200_block_wcc_min(case.handle, case.blk, vl, vc, C.byref(case.err))
    else:
        dist = torch.zeros(case.n_span, dtype=case.tt, device="cuda")
        cand = torch.empty(case.n_span, dtype=torch.int64, device="cuda")
        vd, vc = case.view(dist, case.tid), case.view(cand, 3)
        code = lib.cugraph_b200_block_sssp_relax(case.handle, case.blk, vd, 1e30, case.n_span, 1, 0, vc, C.byref(case.err))
    assert code == 0, lib.cugraph_error_message(case.err)
    torch.cuda.synchronize()


def pull_entries_agree(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, label):
    """cugraph_b200_block_sweep(transposed = FALSE, use_weights = TRUE) against cugraph_b200_block_pull_sweep: the same
    x, two y arrays, both within the bound and within twice the bound of each other.  A block remembers one y per
    orientation, so alternating between the two arrays makes every sweep write every row (0 in the empty ones)"""
    case = Case(lib, monkeypatch, capfd, rows, cols, w, n_rows, n_cols, dtype, knobs, l2_bytes, label)
    try:
        for k, alpha in enumerate(sr.ALPHAS):
            state = case.rng.bit_generator.state
            y1, x1 = case.sweep("a", False, True, alpha, entry="pull_sweep")
            case.rng.bit_generator.state = state
            y2, x2 = case.sweep("b", False, True, alpha)
            assert np.array_equal(x1, x2, equal_nan=True)
            case.check(y1, x1, False, True, alpha, 0, f"{label} block_pull_sweep")
            case.check(y2, x2, False, True, alpha, 0, f"{label} block_sweep")
            A, deg, read, _ = case.orientation(False, True)
            S = abs(alpha) * (abs(A) @ np.abs(np.where(read, x1[:case.n_span].astype(np.float64), 0.0)))
            assert np.all(np.abs(y1 - y2) <= 4.0 * (S * (4.0 * case.u + deg * 2.0 ** -52)) + 2 * case.u * np.abs(y1)), label
    finally:
        case.free()
