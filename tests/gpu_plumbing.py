"""Plumbing the GPU tests share: the default renderer, device copies, device-error readers, a context with a small host
pipeline budget and a thread pool for float64 references.  Test infrastructure."""
import contextlib
import ctypes
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch


def to(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _R():
    from sonicsim_b200 import render
    return render, render.default_renderer()


def _lib():
    from sonicsim_b200 import _lib as L, render
    return L, render.default_renderer()


@contextlib.contextmanager
def small_host_budget_context():
    """A context of its own whose host pipeline budget is 1 MB (SS_HOST_CHUNK_MB is read by ss_create)."""
    L, R = _lib()
    old = os.environ.get("SS_HOST_CHUNK_MB")
    os.environ["SS_HOST_CHUNK_MB"] = "1"
    ctx = ctypes.c_void_p()
    try:
        assert R.lib.ss_create(R.device, ctypes.byref(ctx)) == 0
    finally:
        if old is None:
            del os.environ["SS_HOST_CHUNK_MB"]
        else:
            os.environ["SS_HOST_CHUNK_MB"] = old
    try:
        yield ctx
    finally:
        R.lib.ss_destroy(ctx)


def _rms(v):
    return float(np.sqrt(np.mean(np.square(np.asarray(v, np.float64)))))


def _workers():
    return max(1, min(16, os.cpu_count() or 1))


def pmap(fn, jobs):
    """fn over jobs on a thread pool (the float64 FFTs release the GIL); exceptions propagate."""
    with ThreadPoolExecutor(_workers()) as ex:
        return list(ex.map(fn, jobs))


def _device_errors(R):
    bits = ctypes.c_uint32()
    assert R.lib.ss_device_errors(R.ctx, ctypes.byref(bits)) == 0
    return bits.value


def _error_bits():
    L_, R = _lib()
    bits = ctypes.c_uint32()
    L_.check(R.lib.ss_device_errors(R.ctx, ctypes.byref(bits)))
    return bits.value


def _errors(R):
    try:
        R.check_device_errors()
    except (IndexError, ValueError) as e:
        return type(e), str(e)
    return None


def renderer():
    from sonicsim_b200 import render
    return render.default_renderer()


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
