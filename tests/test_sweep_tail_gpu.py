"""The piece-stream sweep with a tail on the GPU: the rows of in-degree < 8 leave the stream and are swept by k_sweep_tail
after the bands, from the tail layout (runs of equal in-degree, lane-interleaved ids, work units drawn from a cursor).  A
forced bound on RMAT-16 (the default gives such a small graph no tail), with one band and with three, against the fp64 oracle
(1e-6 relative at equal iteration count) and row by row against the plain sweep.  Every bound, element type and layout path
is checked row by row against an fp64 reference in tests/test_sweep_rows_gpu.py."""
import ctypes as C

import numpy as np
import pytest

import oracle
from oracle.rmat import rmat_edgelist
from tests.gpu_util import by_vertex, make_graph
from tests.test_pagerank_gpu import REL, _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("bands,weighted", [("0", False), ("3", False), ("3", True)])
def test_forced_tail_piece_stream_vs_oracle(monkeypatch, bands, weighted):
    from cugraph_b200 import _capi
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_MIN_EDGES", "0")      # read when the handle is created (make_graph does)
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_TAIL_DEGREE", "8")
    monkeypatch.setenv("CUGRAPH_B200_SWEEP_BANDS", bands)
    scale = 16
    s, d = rmat_edgelist(scale, 16 << scale, seed=300 + scale)
    w = np.random.default_rng(8).random(s.shape[0]).astype(np.float32) + 0.25 if weighted else None
    V = 1 << scale
    h, g = make_graph(s, d, w, store_transposed=True, vertices=np.arange(V, dtype=np.int32))
    verts, vals, conv = _run(h, g, 0.85, 0.0, 30)
    ref, _, _ = oracle.pagerank(s, d, V, None if w is None else w.astype(np.float64), alpha=0.85, epsilon=0.0, max_iterations=30)
    np.testing.assert_allclose(by_vertex(verts, vals, V), ref, rtol=REL, atol=1e-12)
    out = (C.c_double * 8)()
    err = C.c_void_p()
    f = _capi.lib().cugraph_b200_debug_compare_sweeps
    f.restype = C.c_int
    f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p)]
    _capi.check(f(h.ptr, g.ptr, C.cast(out, C.c_void_p), C.byref(err)), err, "cugraph_b200_debug_compare_sweeps")
    assert out[0] < 2e-6 and out[4] < 2e-6 and out[3] == 0 and out[7] == 0, list(out)
