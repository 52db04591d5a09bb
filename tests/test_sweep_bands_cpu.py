"""Row bands of the piece stream (sweep_layout.cu, sweep.cuh): the covered rows are split into bands whose fp64 accumulators
fit in the L2, pieces are ordered by (band, block, kind) and the sweep runs band after band.  Checked on the CPU: the
banded layout holds every (row, source[, weight]) exactly once, a band's chunks hold only its rows, each band's CTA ranges
partition its phases, the planner lays bands out one after the other, and PageRank through the emulated kernels matches the
oracle for forced band counts."""
import ctypes as C

import numpy as np
import pytest

import oracle
from cugraph_b200 import _capi
from tests.test_emu_algorithms_cpu import dense_ids, run_pagerank
from tests.test_emu_staging_cpu import check_sweep_layout, create_graph, emu, make_edges, primary  # noqa: F401
from tests.test_sweep_plan_cpu import CHUNK_GROUPS, KINDS, PIECES, STEPS


def bands_of(L, g, es, n_cta_flat):
    L.emu_sweep_bands.restype = C.c_int
    L.emu_sweep_bands.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    cap = 4096
    n_cta = C.c_int()
    band_row = np.zeros(cap, dtype=np.int32)
    band_phase = np.zeros(cap, dtype=np.int32)
    n_bands = L.emu_sweep_bands(g, es, C.byref(n_cta), band_row.ctypes.data, band_phase.ctypes.data, cap)
    assert n_bands >= 1 and n_bands * n_cta.value == n_cta_flat
    return n_bands, n_cta.value, band_row[:n_bands + 1], band_phase[:n_bands + 1]


def layout_arrays(L, g):
    ints = (C.c_int64 * 12)()
    ptrs = (C.c_void_p * 6)()
    assert L.emu_sweep_layout(C.c_void_p(L.handle), g, ints, ptrs) == 0
    n_rs, n_chunks, n_phases, n_cta_flat, es = int(ints[5]), int(ints[6]), int(ints[7]), int(ints[8]), int(ints[10])
    as_np = lambda p, n: np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_int32)), shape=(n,)).copy()
    return dict(rows=as_np(ptrs[2], n_rs), chunks=as_np(ptrs[3], 4 * n_chunks).reshape(-1, 4),
                phases=as_np(ptrs[4], 4 * n_phases).reshape(-1, 4), cta=as_np(ptrs[5], n_cta_flat + 1), n_cta_flat=n_cta_flat,
                es=es)


@pytest.mark.parametrize("bands,weighted", [("0", False), ("3", False), ("7", True), ("100000", False)])
def test_banded_layout(emu, monkeypatch, bands, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_BANDS", bands)
    src, dst, w = make_edges(120_000, 900_000, seed=5 + weighted, weighted=weighted, id_offset=11)
    g = create_graph(emu, src, dst, w)
    P = primary(emu, g)
    check_sweep_layout(emu, g, P)                       # every (row, source[, weight]) exactly once
    A = layout_arrays(emu, g)
    n_bands, n_cta, band_row, band_phase = bands_of(emu, g, A["es"], A["n_cta_flat"])
    n_cov = P["seg"][5]
    assert band_row[0] == 0 and band_row[-1] == n_cov and (np.diff(band_row) > 0).all()
    assert (band_row[:-1] % 512 == 0).all()             # the finish kernel's spans never straddle a band bound
    asked = int(bands) or -(-(n_cov * 8 * 2) // (1 << 20))   # default: a band's accumulators take half of the L2 (1 MB emulated)
    asked = min(asked, -(-n_cov // 512))
    band_rows = -(-(-(-n_cov // asked)) // 512) * 512
    assert n_bands == -(-n_cov // band_rows) and n_bands > 1
    if bands not in ("0", "100000"):
        assert n_bands == int(bands)
    rows, chunks, phases, cta = A["rows"], A["chunks"], A["phases"], A["cta"]
    assert band_phase[0] == 0 and band_phase[-1] == len(phases) and (np.diff(band_phase) > 0).all()
    for b in range(n_bands):
        lo, hi = int(band_phase[b]), int(band_phase[b + 1])
        # the CTA ranges of band b partition exactly its phases
        own = cta[b * n_cta: (b + 1) * n_cta + 1]
        assert own[0] == lo and own[-1] == hi and (np.diff(own) >= 0).all()
        # every chunk of band b holds only rows of band b
        for c0 in range(phases[lo][1], phases[hi - 1][2]):
            _, row0, n_groups, kind = chunks[c0]
            r = rows[row0: row0 + n_groups * PIECES[kind]]
            r = r[r >= 0]
            assert r.size and (r >= band_row[b]).all() and (r < band_row[b + 1]).all(), (b, c0)
    emu.cugraph_graph_free(g)


@pytest.mark.parametrize("bands", [2, 3, 7])
@pytest.mark.parametrize("weighted", [False, True])
def test_pagerank_forced_bands_emulated(emu, monkeypatch, bands, weighted):  # noqa: F811
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_BANDS", str(bands))
    src, dst, w = make_edges(60_000, 250_000, seed=71 + bands, weighted=weighted, id_offset=2)
    g = create_graph(emu, src, dst, w)
    verts, pr, it = run_pagerank(emu, g, 0.85, 0.0, 20)
    A = layout_arrays(emu, g)
    assert bands_of(emu, g, A["es"], A["n_cta_flat"])[0] == bands
    ids, s, d = dense_ids(src, dst)
    ref, _, _ = oracle.pagerank(s, d, ids.size, None if w is None else w.astype(np.float64), alpha=0.85, epsilon=0.0,
                                max_iterations=20)
    assert it == 20
    got = np.zeros(ids.size)
    got[np.searchsorted(ids, verts)] = pr
    np.testing.assert_allclose(got, ref, rtol=1e-6, atol=0)
    emu.cugraph_graph_free(g)


def plan_bands(counts, sm_count):
    """counts[band][b][k] pieces of kind k in block b of the band"""
    L = _capi.lib()
    counts = np.asarray(counts, dtype=np.int64)
    n_bands, B = counts.shape[:2]
    cstart = np.zeros(n_bands * B * KINDS + 1, dtype=np.int32)
    cstart[1:] = np.cumsum(counts.reshape(-1))
    cap = int(sum(-(-int(c) // PIECES[k]) for c, k in zip(counts.reshape(-1), np.tile(np.arange(KINDS), n_bands * B)))) + 8
    totals = (C.c_int64 * 3)()
    chunks = np.zeros((cap, 4), dtype=np.int32)
    fills = np.zeros((cap, 4), dtype=np.int32)
    phases = np.zeros((cap + n_bands * sm_count, 4), dtype=np.int32)
    cta = np.zeros(n_bands * sm_count + 1, dtype=np.int32)
    band_phase = np.zeros(n_bands + 1, dtype=np.int32)
    n_chunks, n_phases, err = C.c_size_t(), C.c_size_t(), C.c_void_p()
    f = L.cugraph_b200_debug_plan_sweep_bands
    f.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                  C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    code = f(cstart.ctypes.data, n_bands, B, sm_count, totals, chunks.ctypes.data, fills.ctypes.data, cap, C.byref(n_chunks),
             phases.ctypes.data, phases.shape[0], C.byref(n_phases), cta.ctypes.data, cta.size, band_phase.ctypes.data,
             C.byref(err))
    _capi.check(code, err, "cugraph_b200_debug_plan_sweep_bands")
    n_cta = int(totals[2])
    return dict(steprows=int(totals[0]), rowslots=int(totals[1]), n_cta=n_cta, chunks=chunks[:n_chunks.value],
                fills=fills[:n_chunks.value], phases=phases[:n_phases.value], cta=cta[:n_bands * n_cta + 1],
                band_phase=band_phase, cstart=cstart)


def test_plan_bands():
    r = np.random.default_rng(1)
    n_bands, B = 4, 12
    counts = np.zeros((n_bands, B, KINDS), dtype=np.int64)
    for band in range(n_bands):                          # band 0 holds the hubs: few, long pieces; later bands many short ones
        for b in range(B):
            shape = np.array([1, 1, 1, 2, 2, 2, 2, 2, 2, 2, 30]) if band == 0 else np.array([40, 12, 8, 4, 2, 1, .5, .3, .2, .1, 0])
            counts[band, b] = (3000 / (1 + b) * shape * r.uniform(0.5, 1.5, KINDS)).astype(np.int64)
    counts[2, 5] = 0                                     # an empty (band, block)
    P = plan_bands(counts, 132)
    chunks, fills, phases, cta, bp, n_cta = P["chunks"], P["fills"], P["phases"], P["cta"], P["band_phase"], P["n_cta"]
    # chunks tile the step-row / row-slot spaces in order; each one's pieces are one (band, block, kind) run
    sr = rs = 0
    band_of_chunk = np.zeros(len(chunks), dtype=np.int64)
    for i, ((sr0, row0, g, kind), (p0, p1, blk, _)) in enumerate(zip(chunks, fills)):
        assert sr0 == sr and row0 == rs and 1 <= g <= CHUNK_GROUPS[kind]
        sr += g * STEPS[kind]
        rs += g * PIECES[kind]
        key = int(np.searchsorted(P["cstart"], p0, side="right")) - 1
        while P["cstart"][key + 1] == P["cstart"][key]:  # skip empty keys at p0
            key += 1
        assert key % KINDS == kind and (key // KINDS) % B == blk and P["cstart"][key + 1] == p1
        band_of_chunk[i] = key // KINDS // B
    assert sr == P["steprows"] and rs == P["rowslots"]
    assert (np.diff(band_of_chunk) >= 0).all()           # bands one after the other
    assert n_cta == min(132, int(np.bincount(band_of_chunk).max()))
    for band in range(n_bands):
        groups = sum(int(c[2]) for c, bb in zip(chunks, band_of_chunk) if bb == band)
        assert groups == sum(-(-int(c) // PIECES[k]) for b in range(B) for k, c in enumerate(counts[band, b]))
    # the phases of band b are [bp[b], bp[b+1]), their chunks are the band's, and its CTA ranges partition them
    assert bp[0] == 0 and bp[-1] == len(phases) and len(cta) == n_bands * n_cta + 1
    at = 0
    for blk, c0, c1, _ in phases:
        assert c0 == at and c1 > c0 and (fills[c0:c1, 2] == blk).all()
        at = c1
    assert at == len(chunks)
    for band in range(n_bands):
        ph = phases[bp[band]:bp[band + 1]]
        assert (band_of_chunk[ph[:, 1]] == band).all() and (band_of_chunk[ph[:, 2] - 1] == band).all()
        own = cta[band * n_cta:(band + 1) * n_cta + 1]
        assert own[0] == bp[band] and own[-1] == bp[band + 1] and (np.diff(own) >= 0).all()
        for c in range(n_cta):                          # a block shows up at most once per CTA range
            blks = phases[own[c]:own[c + 1], 0]
            assert len(set(blks.tolist())) == len(blks)


def test_plan_one_band_is_the_single_band_planner():
    from tests.test_sweep_plan_cpu import plan
    r = np.random.default_rng(2)
    counts = (r.random((9, KINDS)) * 5000).astype(np.int64)
    a, b = plan(counts, 132), plan_bands(counts[None], 132)
    for k in ("steprows", "rowslots", "n_cta"):
        assert a[k] == b[k]
    for k in ("chunks", "fills", "phases", "cta"):
        assert np.array_equal(a[k], b[k]), k
    assert list(b["band_phase"]) == [0, len(b["phases"])]
