"""Host-side planner of the shared-memory pull sweep (sweep_layout.cu: plan_sweep, reached through the C ABI debug hook
cugraph_b200_debug_plan_sweep): groups -> chunks -> per-CTA ranges -> phases, from the piece counts per (block, kind)
alone.  Pure host code, so the structure the GPU kernel relies on is checkable here."""
import ctypes as C

import numpy as np
import pytest

from cugraph_b200 import _capi

KINDS = 11
PIECES = [256, 128, 64] + [32] * 8          # pieces per group of kind S, Q, H, F1..F8
STEPS = [1, 1, 1] + list(range(1, 9))       # step-rows per group
CHUNK_GROUPS = [2, 4, 4, 6, 3, 2, 2, 1, 1, 1, 1]


def plan(counts, sm_count):
    """counts[b][k] pieces of kind k in block b"""
    L = _capi.lib()
    counts = np.asarray(counts, dtype=np.int64)
    B = counts.shape[0]
    cstart = np.zeros(B * KINDS + 1, dtype=np.int32)
    cstart[1:] = np.cumsum(counts.reshape(-1))
    cap = int(sum(-(-int(c) // (PIECES[k] * 1)) for row in counts for k, c in enumerate(row))) + 8
    totals = (C.c_int64 * 3)()
    chunks = np.zeros((cap, 4), dtype=np.int32)
    fills = np.zeros((cap, 4), dtype=np.int32)
    phases = np.zeros((cap + sm_count, 4), dtype=np.int32)
    cta = np.zeros(sm_count + 1, dtype=np.int32)
    n_chunks, n_phases, err = C.c_size_t(), C.c_size_t(), C.c_void_p()
    L.cugraph_b200_debug_plan_sweep.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                                C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    code = L.cugraph_b200_debug_plan_sweep(cstart.ctypes.data, B, sm_count, totals, chunks.ctypes.data, fills.ctypes.data, cap,
                                           C.byref(n_chunks), phases.ctypes.data, cap + sm_count, C.byref(n_phases),
                                           cta.ctypes.data, sm_count + 1, C.byref(err))
    _capi.check(code, err, "cugraph_b200_debug_plan_sweep")
    n_cta = int(totals[2])
    return dict(steprows=int(totals[0]), rowslots=int(totals[1]), n_cta=n_cta, chunks=chunks[:n_chunks.value],
                fills=fills[:n_chunks.value], phases=phases[:n_phases.value], cta=cta[:n_cta + 1], cstart=cstart)


def check(P, counts):
    counts = np.asarray(counts)
    chunks, fills, phases, cta = P["chunks"], P["fills"], P["phases"], P["cta"]
    # chunks tile the step-row and row-slot spaces in order, one kind and one block each, at most the kind's group count
    sr = rs = 0
    for (sr0, row0, g, kind), (p0, p1, blk, _) in zip(chunks, fills):
        assert sr0 == sr and row0 == rs and 1 <= g <= CHUNK_GROUPS[kind]
        assert row0 % 32 == 0
        sr += g * STEPS[kind]
        rs += g * PIECES[kind]
        key = blk * KINDS + kind
        assert P["cstart"][key] <= p0 < p1 == P["cstart"][key + 1]
        assert (p0 - P["cstart"][key]) % PIECES[kind] == 0
    assert sr == P["steprows"] and rs == P["rowslots"]
    # every (block, kind) run is covered exactly: groups = ceil(pieces / pieces-per-group)
    for b in range(counts.shape[0]):
        for k in range(KINDS):
            groups = int(sum(c[2] for c, f in zip(chunks, fills) if f[2] == b and c[3] == k))
            assert groups == -(-int(counts[b, k]) // PIECES[k])
    # phases: contiguous chunk ranges of one block, consecutive, covering all chunks; CTA ranges contiguous over the phases
    at = 0
    for blk, c0, c1, _ in phases:
        assert c0 == at and c1 > c0 and (fills[c0:c1, 2] == blk).all()
        at = c1
    assert at == len(chunks)
    assert cta[0] == 0 and cta[-1] == len(phases) and (np.diff(cta) >= 0).all()
    # a block shows up at most once per CTA range
    for c in range(P["n_cta"]):
        blks = phases[cta[c]:cta[c + 1], 0]
        assert len(set(blks.tolist())) == len(blks)


def test_plan_power_law_blocks():
    r = np.random.default_rng(0)
    B = 40
    counts = np.zeros((B, KINDS), dtype=np.int64)
    for b in range(B):
        scale = 200000 / (1 + b) ** 1.3
        counts[b] = (scale * np.array([6, 2, 1.5, 1, .6, .3, .2, .1, .05, .05, 1.0 if b == 0 else 0.02]) * r.uniform(0.5, 1.5, KINDS)).astype(np.int64)
    P = plan(counts, 148)
    check(P, counts)
    assert P["n_cta"] == 148
    # balance: the estimated cost per CTA range is within 25 % of the mean (chunk granularity + per-block overhead)
    cost = lambda g, k: g * (STEPS[k] * 14.0 + PIECES[k] * (0.1 if k == 10 else 1.2) + 4.0)
    per = []
    for c in range(148):
        c0, c1 = P["phases"][P["cta"][c]][1], P["phases"][P["cta"][c + 1] - 1][2]
        per.append(sum(cost(g, k) for _, _, g, k in P["chunks"][c0:c1]) + 2500.0 * (P["cta"][c + 1] - P["cta"][c]))
    per = np.array(per)
    assert per.max() < 1.25 * per.mean(), (per.max(), per.mean())


def test_plan_tiny_and_empty_kinds():
    counts = np.zeros((3, KINDS), dtype=np.int64)
    counts[0, 0] = 1          # one S piece
    counts[2, 10] = 33        # two F8 groups
    P = plan(counts, 148)
    check(P, counts)
    assert P["n_cta"] == len(P["chunks"]) == 3 and len(P["phases"]) in (2, 3)   # a range may stay empty: its CTA steals


def test_plan_single_cta():
    counts = np.full((5, KINDS), 700, dtype=np.int64)
    P = plan(counts, 1)
    check(P, counts)
    assert P["n_cta"] == 1 and len(P["phases"]) == 5
