"""Synthetic inputs for tests and bench: the RMAT edge list comes from the library's device generator
(cugraph_b200_generate_rmat_edgelist, csrc/generators.cu — the reference's sampling rule, clip-and-flip and id scramble,
cpp/src/generators/generate_rmat_edgelist.cuh:66-108, scramble.cuh:44-67, over a counter-based uniform stream);
oracle/rmat.py:rmat_edgelist_counter is its numpy twin (bit-exact, tests/test_generators_*.py)."""
from __future__ import annotations

import ctypes as C


def rmat_edgelist(scale: int, num_edges: int, a=0.57, b=0.19, c=0.19, seed=0, scramble_ids=True, clip_and_flip=False,
                  device="cuda", handle=None, first_edge=0):
    """(src, dst) int32 CUDA tensors of `num_edges` RMAT edges over 2**scale vertices: edges [first_edge, first_edge +
    num_edges) of the stream of `seed`, so that consecutive slices concatenate to the output of one call over their union."""
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    # a handle on torch's current stream: the generator kernel is ordered with the caller's torch work on both sides
    h = handle or ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
    src = torch.empty(num_edges, dtype=torch.int32, device=device)
    dst = torch.empty(num_edges, dtype=torch.int32, device=device)
    vs, vd, err = View(src), View(dst), C.c_void_p()
    h.order_after_caller()
    code = L.cugraph_b200_generate_rmat_edgelist_at(h.ptr, int(scale), int(first_edge), int(num_edges), float(a), float(b),
                                                    float(c), int(seed), 1 if clip_and_flip else 0, 1 if scramble_ids else 0,
                                                    vs.ptr, vd.ptr, C.byref(err))
    vs.free()
    vd.free()
    _capi.check(code, err, "cugraph_b200_generate_rmat_edgelist_at")
    if handle is not None:
        torch.cuda.synchronize()  # a caller-supplied handle may run on its own stream
    return src, dst


def uniform_values(n: int, seed: int, lo: float, hi: float, dtype=None, device="cuda", handle=None, first=0):
    """`n` values of the counter-based uniform stream of `seed` (cugraph_b200_generate_uniform_at): values [first, first + n),
    in [lo, hi), float32 (default), float64 or int32."""
    import torch
    from cugraph_b200 import _capi
    from cugraph_b200.pylibcugraph.resource_handle import ResourceHandle
    from cugraph_b200.pylibcugraph.utils import View
    L = _capi.lib()
    h = handle or ResourceHandle(stream=torch.cuda.current_stream().cuda_stream)
    out = torch.empty(n, dtype=dtype or torch.float32, device=device)
    vo, err = View(out), C.c_void_p()
    h.order_after_caller()
    code = L.cugraph_b200_generate_uniform_at(h.ptr, int(seed), int(first), float(lo), float(hi), vo.ptr, C.byref(err))
    vo.free()
    _capi.check(code, err, "cugraph_b200_generate_uniform_at")
    if handle is not None:
        torch.cuda.synchronize()
    return out
