"""Graph staging on the CPU: the real staging code (capi_graph.cu, graph_build.cu, sweep_layout.cu — renumbering, the packed-key sort,
binning, the piece stream of the shared-memory sweep) compiled as plain C++ against
the host emulation shim in emu/ and driven through the real C ABI with numpy arrays.  The staging kernels are
data-parallel loops without intra-block communication, so executing every "thread" of a launch in turn is exact.

Checked against numpy: the stored graph is the input multigraph (external ids), rows are degree-descending with sorted
neighbours and correct segment bounds; the piece stream reproduces every (row, source[, weight]) of every non-empty row
exactly once, padding only where allowed.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INT32, INT64, FLOAT32, FLOAT64 = 2, 3, 8, 9


@pytest.fixture(scope="module")
def emu():
    sys.path.insert(0, os.path.join(ROOT, "emu"))
    import build_emu
    try:
        path = build_emu.build()
    except Exception as e:  # no host compiler: nothing to emulate with
        pytest.skip(f"emulation build unavailable: {e}")
    L = C.CDLL(path)
    L.cugraph_create_resource_handle.restype = C.c_void_p
    L.cugraph_create_resource_handle.argtypes = [C.c_void_p]
    L.cugraph_type_erased_device_array_view_create.restype = C.c_void_p
    L.cugraph_type_erased_device_array_view_create.argtypes = [C.c_void_p, C.c_size_t, C.c_int]
    L.cugraph_type_erased_device_array_view_free.argtypes = [C.c_void_p]
    L.cugraph_error_message.restype = C.c_char_p
    L.cugraph_error_message.argtypes = [C.c_void_p]
    L.cugraph_graph_free.argtypes = [C.c_void_p]
    L.emu_graph_primary.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_sweep_layout.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    L.emu_reload_tuning.argtypes = [C.c_void_p]
    L.handle = L.cugraph_create_resource_handle(None)
    assert L.handle
    return L


class Props(C.Structure):
    _fields_ = [("is_symmetric", C.c_int), ("is_multigraph", C.c_int)]


def make_edges(V, E, seed, weighted=False, id_offset=0):
    """power-law-ish destinations AND sources (hubs on both sides), multi-edges and self-loops included"""
    r = np.random.default_rng(seed)
    dst = np.minimum((V * r.random(E) ** 3.0).astype(np.int64), V - 1)
    src = np.minimum((V * r.random(E) ** 2.0).astype(np.int64), V - 1)
    perm = r.permutation(V)                     # external ids carry no degree information
    src, dst = perm[src] + id_offset, perm[dst] + id_offset
    w = (r.random(E).astype(np.float32) + 0.25) if weighted else None
    return src.astype(np.int32), dst.astype(np.int32), w


def create_graph(L, src, dst, w, **flags):
    L.emu_reload_tuning(C.c_void_p(L.handle))   # the knobs are read from the environment per handle; tests change it per case
    views = [L.cugraph_type_erased_device_array_view_create(a.ctypes.data, a.size, t) if a is not None else None
             for a, t in ((src, INT32), (dst, INT32), (w, FLOAT32))]
    g, err = C.c_void_p(), C.c_void_p()
    code = L.cugraph_graph_create_with_times_sg(
        C.c_void_p(L.handle), C.byref(Props(0, 1)), None, C.c_void_p(views[0]), C.c_void_p(views[1]),
        C.c_void_p(views[2]) if views[2] else None, None, None, None, None,
        int(flags.get("store_transposed", 1)), 1, int(flags.get("drop_self_loops", 0)), int(flags.get("drop_multi_edges", 0)),
        int(flags.get("symmetrize", 0)), 0, C.byref(g), C.byref(err))
    assert code == 0, L.cugraph_error_message(err)
    for v in views:
        if v:
            L.cugraph_type_erased_device_array_view_free(v)
    return g


def as_np(ptr, n, dtype):
    if not ptr or n == 0:
        return np.zeros(0, dtype=dtype)
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(int(n),))


def primary(L, g):
    ints = (C.c_int64 * 8)()
    seg = (C.c_int32 * 8)()
    ptrs = (C.c_void_p * 5)()
    assert L.emu_graph_primary(g, ints, seg, ptrs) == 0
    n_rows, nnz, offs64, nnz_hi, nv, weighted, wsize = [int(x) for x in ints[:7]]
    off = as_np(ptrs[0], n_rows + 1, np.int64 if offs64 else np.int32)
    idx = as_np(ptrs[1], nnz, np.int32)
    w = as_np(ptrs[2], nnz, np.float32 if wsize == 4 else np.float64) if weighted else None
    ext = as_np(ptrs[3], nv, np.int32)
    return dict(n_rows=n_rows, nnz=nnz, nnz_hi=nnz_hi, nv=nv, off=off, idx=idx, w=w, ext=ext, seg=list(seg), offs64=bool(offs64))


def check_csr(P, src, dst, w):
    off, idx, ext = P["off"], P["idx"], P["ext"]
    deg = np.diff(off)
    assert (deg[:-1] >= deg[1:]).all()                                  # degree-descending rows = the binning
    for k, t in enumerate((32, 16, 8, 4, 2, 1, 0)):
        assert P["seg"][k] == int((deg >= t).sum())
    assert P["nnz_hi"] == int(off[P["seg"][0]])
    rows = np.repeat(np.arange(P["n_rows"]), deg)
    same_row = rows[1:] == rows[:-1]
    assert (idx[1:][same_row] >= idx[:-1][same_row]).all()               # neighbours ascending inside a row
    # the stored graph is the input multigraph (rows = destinations, entries = sources), on external ids
    got = np.stack([ext[rows], ext[idx]], 1)
    exp = np.stack([dst, src], 1)
    if w is None:
        key = lambda a: a[np.lexsort((a[:, 1], a[:, 0]))]
        assert (key(got) == key(exp)).all()
    else:
        o1 = np.lexsort((P["w"], got[:, 1], got[:, 0]))
        o2 = np.lexsort((w, exp[:, 1], exp[:, 0]))
        assert (got[o1] == exp[o2]).all() and (P["w"][o1] == w[o2]).all()
    assert sorted(set(ext.tolist())) == sorted(set(src.tolist()) | set(dst.tolist()))


def lds_wavefronts(ids):
    """shared-memory wavefronts of one warp-wide 4-byte gather: max over the 32 banks of the distinct addresses on a bank"""
    u = np.unique(ids)
    return int(np.bincount(u & 31, minlength=32).max())


KIND_PIECES = [256, 128, 64] + [32] * 8     # pieces per group: S, Q, H, F1..F8
KIND_STEPS = [1, 1, 1] + list(range(1, 9))  # step-rows per group


def red_units(rr, stats):
    """rr[k, lane] = rows of the 32 lanes of one warp-wide accumulation (-1 = lane idle): counts the units, the 32-byte
    sectors of the fp64 accumulators they touch (4 rows each) and the units whose lanes hold 32 consecutive rows"""
    for unit in rr:
        live = unit[unit >= 0]
        if live.size == 0:
            continue
        stats["red_units"] = stats.get("red_units", 0) + 1
        stats["red_lanes"] = stats.get("red_lanes", 0) + int(live.size)
        stats["red_sectors"] = stats.get("red_sectors", 0) + int(np.unique(live >> 2).size)
        base = int(live[0]) - int(np.flatnonzero(unit >= 0)[0])
        if base % 32 == 0 and (unit[unit >= 0] == base + np.flatnonzero(unit >= 0)).all():
            stats["aligned_units"] = stats.get("aligned_units", 0) + 1
            stats["aligned_lanes"] = stats.get("aligned_lanes", 0) + int(live.size)


def sweep_pieces(L, g, P, stats=None):
    """(row, col[, w]) triples reconstructed from the piece stream + structural checks.
    stats: dict that receives the LDS count and the wavefront count of the F kinds (bank order)."""
    ints = (C.c_int64 * 12)()
    ptrs = (C.c_void_p * 6)()
    rc = L.emu_sweep_layout(C.c_void_p(L.handle), g, ints, ptrs)
    assert rc == 0, f"emu_sweep_layout returned {rc}"
    W, B, n_cov, nnz, n_sr, n_rs, n_chunks, n_phases, n_cta, bank, es, n_pieces = [int(x) for x in ints[:12]]
    assert n_cov == P["seg"][5] and nnz == P["nnz"]          # every non-empty row, every edge
    ids = as_np(ptrs[0], n_sr * 32 * 8, np.uint16).reshape(n_sr, 32, 8)
    sw = as_np(ptrs[1], n_sr * 32 * 8, np.float32).reshape(n_sr, 32, 8) if P["w"] is not None else None
    rows = as_np(ptrs[2], n_rs, np.int32)
    chunks = as_np(ptrs[3], 4 * n_chunks, np.int32).reshape(-1, 4)
    phases = as_np(ptrs[4], 4 * n_phases, np.int32).reshape(-1, 4)
    cta = as_np(ptrs[5], n_cta + 1, np.int32)
    assert cta[0] == 0 and cta[-1] == n_phases and (np.diff(cta) >= 0).all()
    blk_of_chunk = np.zeros(n_chunks, dtype=np.int64)
    at = 0
    for blk, c0, c1, _ in phases:
        assert c0 == at and c1 > c0
        blk_of_chunk[c0:c1] = blk
        at = c1
    assert at == n_chunks
    out_r, out_c, out_w = [], [], []
    n_real_pieces = 0
    for ci, (sr0, row0, n_groups, kind) in enumerate(chunks):
        blk = int(blk_of_chunk[ci])
        steps, ppg = KIND_STEPS[kind], KIND_PIECES[kind]
        for q in range(n_groups):
            if kind < 3:      # S / Q / H: R pieces of E entries per lane
                R = ppg // 32
                E = 8 // R
                sl = ids[sr0 + q].astype(np.int64).reshape(32, R, E)
                rr = rows[row0 + q * ppg: row0 + (q + 1) * ppg].reshape(32, R)
                real = sl < W
                assert (sl <= W).all()                              # narrow kinds pad with column W only
                assert (real[:, :, :-1] >= real[:, :, 1:]).all()    # padding behind the real entries of a piece
                assert not real[rr < 0].any()                       # unused pieces are all padding
                assert (real.sum(2)[rr >= 0] >= 1).all()
                n_real_pieces += int((rr >= 0).sum())
                if stats is not None:   # piece slot k * 32 + lane of the group = the lanes of the k-th RED of the step
                    red_units(rr.T, stats)
                cols = sl + blk * W
                out_r.append(np.repeat(rr[:, :, None], E, 2)[real]); out_c.append(cols[real])
                if sw is not None:
                    ww = sw[sr0 + q].reshape(32, R, E)
                    assert (ww[~real] == 0).all()
                    out_w.append(ww[real])
            else:
                sl = ids[sr0 + q * steps: sr0 + (q + 1) * steps].astype(np.int64)   # [steps, 32 lanes, 8]
                rr = rows[row0 + q * 32: row0 + (q + 1) * 32]
                assert (sl < W + 64).all()                          # padding = one of the slice's zero columns
                real = sl < W
                assert not real[:, rr < 0, :].any()
                per_piece = real.sum((0, 2))
                assert (per_piece[rr >= 0] > (steps - 1) * 8).all() and (per_piece[rr >= 0] <= steps * 8).all()   # the kind fits
                if not bank:
                    flat = real.transpose(1, 0, 2).reshape(32, -1)
                    assert (flat[:, :-1] >= flat[:, 1:]).all()
                n_real_pieces += int((rr >= 0).sum())
                if stats is not None:
                    red_units(rr[None, :], stats)
                    stats["lds"] = stats.get("lds", 0) + 8 * steps
                    stats["wavefronts"] = stats.get("wavefronts", 0) + sum(lds_wavefronts(sl[j, :, k]) for j in range(steps) for k in range(8))
                cols = sl + blk * W
                r3 = np.broadcast_to(rr[None, :, None], sl.shape)
                out_r.append(r3[real]); out_c.append(cols[real])
                if sw is not None:
                    ww = sw[sr0 + q * steps: sr0 + (q + 1) * steps]
                    assert (ww[~real] == 0).all()
                    out_w.append(ww[real])
    assert n_real_pieces == n_pieces
    r = np.concatenate(out_r) if out_r else np.zeros(0, np.int64)
    c = np.concatenate(out_c) if out_c else np.zeros(0, np.int64)
    w = np.concatenate(out_w) if out_w else None
    return dict(r=r, c=c, w=w, W=W, B=B, chunks=chunks, phases=phases, bank=bank)


def check_sweep_layout(L, g, P, stats=None):
    H = sweep_pieces(L, g, P, stats)
    n_cov, nnz = P["seg"][5], P["nnz"]
    rows = np.repeat(np.arange(n_cov), np.diff(P["off"][:n_cov + 1]))
    cols = P["idx"][:nnz].astype(np.int64)
    assert H["r"].size == nnz
    if P["w"] is None:
        o1, o2 = np.lexsort((H["c"], H["r"])), np.lexsort((cols, rows))
        assert (H["r"][o1] == rows[o2]).all() and (H["c"][o1] == cols[o2]).all()
    else:
        o1, o2 = np.lexsort((H["w"], H["c"], H["r"])), np.lexsort((P["w"][:nnz], cols, rows))
        assert (H["r"][o1] == rows[o2]).all() and (H["c"][o1] == cols[o2]).all() and (H["w"][o1] == P["w"][:nnz][o2]).all()
    return H


@pytest.mark.parametrize("weighted", [False, True])
def test_staging_and_piece_stream(emu, monkeypatch, weighted):
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    src, dst, w = make_edges(120_000, 900_000, seed=3 + weighted, weighted=weighted, id_offset=17)
    g = create_graph(emu, src, dst, w)
    P = primary(emu, g)
    check_csr(P, src, dst, w)
    assert P["seg"][0] > 500                      # there are degree >= 32 rows, and several column blocks
    H = check_sweep_layout(emu, g, P)
    assert H["B"] >= 2 and all((H["chunks"][:, 3] == k).any() for k in (0, 1, 2, 3, 10))   # S, Q, H, F1 and F8 pieces exist
    emu.cugraph_graph_free(g)


@pytest.mark.parametrize("weighted", [False, True])
def test_bank_ordered_slots(emu, monkeypatch, weighted):
    """the F kinds' entries are ordered by shared-memory bank (default for 4-byte values): same (row, source[, weight])
    multiset, and fewer shared-memory wavefronts per gather than the natural order"""
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    src, dst, w = make_edges(120_000, 900_000, seed=21 + weighted, weighted=weighted, id_offset=3)
    res = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("CUGRAPH_B200_SWEEP_BANK_ORDER", mode)
        g = create_graph(emu, src, dst, w)
        P = primary(emu, g)
        st = {}
        H = check_sweep_layout(emu, g, P, stats=st)
        assert H["bank"] == int(mode)
        res[mode] = st["wavefronts"] / st["lds"]
        emu.cugraph_graph_free(g)
    print(f"wavefronts per LDS (F kinds): natural order {res['0']:.3f}, bank order {res['1']:.3f}")
    assert res["1"] < 0.7 * res["0"], res


def test_staging_options(emu, monkeypatch):
    """self-loop / multi-edge removal and symmetrisation against numpy"""
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "1000000000")
    src, dst, _ = make_edges(3_000, 40_000, seed=9)
    g = create_graph(emu, src, dst, None, drop_self_loops=1, drop_multi_edges=1)
    P = primary(emu, g)
    keep = src != dst
    pairs = np.unique(np.stack([dst[keep], src[keep]], 1), axis=0)
    check_csr(P, pairs[:, 1].astype(np.int32), pairs[:, 0].astype(np.int32), None)
    emu.cugraph_graph_free(g)
