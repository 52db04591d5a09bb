"""TEST INFRASTRUCTURE: run the Python surface (cugraph_b200.pylibcugraph, bench.py, scripts/bench_side.py) on a box
without a GPU by pointing `cugraph_b200._capi` at the emulation build of the library (emu/build_emu.py: the CUDA sources
compiled as C++ against a SIMT emulation, "device" memory = host memory) and giving torch's CUDA entry points CPU
stand-ins.  Nothing in the product imports this module; the product library has no CPU path (`_capi.lib()` raises when
libcugraph_c.so is missing).  What this catches: Python-level mistakes in the wrappers and in the measurement scripts
(argument order, result plumbing, JSON assembly) that would otherwise only show on a GPU.  What it cannot
catch: stream ordering, timing, anything about the real kernels' execution."""
import contextlib
import os
import sys
import time

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _FakeStream:
    cuda_stream = 0

    def __init__(self, *a, **k):
        pass

    def synchronize(self):
        pass


class _FakeEvent:
    def __init__(self, enable_timing=False):
        self.t = None

    def record(self, stream=None):
        self.t = time.perf_counter()

    def synchronize(self):
        pass

    def elapsed_time(self, other):
        return (other.t - self.t) * 1e3


def _is_cuda(dev):
    return dev is not None and str(dev).startswith("cuda")


@contextlib.contextmanager
def emulated_python_surface():
    import torch
    sys.path.insert(0, os.path.join(ROOT, "emu"))
    import build_emu
    from cugraph_b200 import _capi
    path = build_emu.build()
    saved = {"lib_path": _capi.LIB_PATH, "lib": _capi._lib}
    _capi.LIB_PATH, _capi._lib = path, None
    patched = []

    def patch(obj, name, new):
        patched.append((obj, name, getattr(obj, name)))
        setattr(obj, name, new)

    def strip_device(fn):
        def wrapper(*a, **k):
            if _is_cuda(k.get("device")):
                k.pop("device")
            return fn(*a, **k)
        return wrapper

    for name in ("empty", "zeros", "ones", "full", "rand", "arange", "tensor", "as_tensor", "randperm", "randint"):
        patch(torch, name, strip_device(getattr(torch, name)))
    real_generator = torch.Generator
    patch(torch, "Generator", lambda device=None: real_generator())
    patch(torch.Tensor, "cuda", lambda self, *a, **k: self)
    patch(torch.Tensor, "pin_memory", lambda self, *a, **k: self)
    real_to = torch.Tensor.to

    def to(self, *a, **k):
        a = tuple(x for x in a if not (isinstance(x, (str, torch.device)) and _is_cuda(x)))
        if _is_cuda(k.get("device")):
            k.pop("device")
        return real_to(self, *a, **k) if (a or k) else self
    patch(torch.Tensor, "to", to)

    def cai(self):
        import numpy as np
        t = self.detach()
        typestr = np.dtype(str(t.dtype).replace("torch.", "")).str
        return {"shape": tuple(t.shape), "typestr": typestr, "data": (t.data_ptr() if t.numel() else 0, False),
                "version": 2, "strides": None if t.is_contiguous() else tuple(s * t.element_size() for s in t.stride())}
    patch(torch.Tensor, "__cuda_array_interface__", property(cai))
    patch(torch.cuda, "is_available", lambda: True)
    patch(torch.cuda, "set_device", lambda *a, **k: None)
    patch(torch.cuda, "synchronize", lambda *a, **k: None)
    patch(torch.cuda, "empty_cache", lambda: None)
    patch(torch.cuda, "current_stream", lambda *a, **k: _FakeStream())
    patch(torch.cuda, "Event", _FakeEvent)
    patch(torch.cuda, "ExternalStream", _FakeStream)
    try:
        yield _capi.lib()
    finally:
        for obj, name, old in reversed(patched):
            setattr(obj, name, old)
        _capi.LIB_PATH, _capi._lib = saved["lib_path"], saved["lib"]


@pytest.fixture(scope="module")
def surface():
    """emulated_python_surface() for the tests of one module; skips them when the emulation cannot be built"""
    pytest.importorskip("torch")
    try:
        cm = emulated_python_surface()
        L = cm.__enter__()
    except Exception as e:  # no host compiler
        pytest.skip(f"emulation build unavailable: {e}")
    yield L
    cm.__exit__(None, None, None)
