"""The device path's two ways of running chunks - ss_render_dev per call, a device plan per run - enqueue the same
chunks: for one batch that spans several chunks and reaches every kind of launch, an ss_render_dev call, a graph run of a
plan and a run of the same plan without a graph (SS_NO_GRAPH) add the same launch count and write the same bits, and
with profiling on, ss_render_dev and the plan time the same number of chunks and still write the same bits."""
import ctypes
import os

import numpy as np
import pytest
import torch

from chunk_budget import chunk_budget  # noqa: F401  (fixture)
from oracle import sonicsim_oracle as so

pytestmark = pytest.mark.gpu

BUDGET = 2 << 20                     # a few sources per chunk: several chunks, forked over the internal streams


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _batch(rng):
    """Sources of every chunk kind, twice over: aligned moving and static (k_render_fast), long RIRs (k_render<LONG>),
    grid-blocked moving (generic k_render), a normalised source with a direct target (k_rir_absmax, k_rir_direct),
    moving sources without bounds_host (k_blocks) and a moving window whose start is read on the device."""
    from sonicsim_b200 import render
    N, T = 48000, 16000
    starts = torch.tensor([0, 5000], dtype=torch.int32, device="cuda")
    srcs, outs, douts = [], [], []

    def moving(P, C, L, host_bounds=True, **kw):
        b = np.linspace(0, N, P).astype(np.int32)
        s = render.MovingSource(_cuda(so.synth_dry(rng, N)), _cuda(so.synth_rirs(rng, P, C, L)), _cuda(b),
                                b if host_bounds else None, **kw)
        rows = T if s.window is not None else N
        srcs.append(s)
        outs.append(torch.full((C, rows), float("nan"), device="cuda"))
        douts.append(torch.full((C, rows), float("nan"), device="cuda") if s.direct_taps else None)

    for k in range(2):
        moving(4, 2, 900)                                               # aligned
        srcs.append(render.StaticSource(_cuda(so.synth_dry(rng, N)), _cuda(so.synth_rirs(rng, 1, 2, 700)[0])))
        outs.append(torch.full((2, N), float("nan"), device="cuda"))
        douts.append(None)
        moving(3, 2, 5000)                                              # long
        moving(40, 1, 1000, host_bounds=False)                          # grid blocking, tables by k_blocks
        moving(4, 2, 900, normalize_rirs=True, direct_taps=40)          # normalised, direct target
        moving(4, 2, 900, host_bounds=False)                            # aligned, tables by k_blocks
        moving(4, 2, 900, window=(starts[k], T))                        # moving window
    return srcs, outs, douts


def _outputs(outs, douts):
    torch.cuda.synchronize()
    return [o.cpu().numpy().copy() for o in outs + [d for d in douts if d is not None]]


def _clear(outs, douts):
    for o in outs + [d for d in douts if d is not None]:
        o.fill_(float("nan"))


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert not np.isnan(x).any() and np.array_equal(x, y)


def test_render_dev_and_plans_run_the_same_chunks(chunk_budget):  # noqa: F811
    from sonicsim_b200 import _lib as L
    R = chunk_budget(BUDGET)
    srcs, outs, douts = _batch(np.random.default_rng(8))
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    c0 = R.launch_count()
    R.render_device(srcs, outs, direct_outs=douts)
    launches = R.launch_count() - c0
    ref = _outputs(outs, douts)

    plan = R.plan_device(srcs, outs, douts)
    plan.run()                                       # captures the graph
    assert plan.is_graph()
    _clear(outs, douts)
    c0 = R.launch_count()
    plan.run()
    assert R.launch_count() - c0 == launches
    _same(ref, _outputs(outs, douts))

    # a context created under SS_NO_GRAPH: the plan enqueues its launches at every run
    os.environ["SS_NO_GRAPH"] = "1"
    ctx2 = ctypes.c_void_p()
    try:
        L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
    finally:
        del os.environ["SS_NO_GRAPH"]
    h = ctypes.c_void_p()
    try:
        L.check(R.lib.ss_set_chunk_bytes(ctx2, BUDGET))
        items, n, keep = R._device_items(srcs, outs, douts)
        L.check(R.lib.ss_plan_create(ctx2, items, n, ctypes.byref(h)))
        _clear(outs, douts)
        c0 = R.lib.ss_launch_count(ctx2)
        L.check(R.lib.ss_plan_run(h, stream))
        assert R.lib.ss_plan_is_graph(h) == 0
        assert R.lib.ss_launch_count(ctx2) - c0 == launches
        _same(ref, _outputs(outs, douts))
    finally:
        if h:
            R.lib.ss_plan_destroy(h)
        R.lib.ss_destroy(ctx2)

    # profiling: chunks one after the other, one timed pair per chunk on both paths
    R.get_profile()
    R.set_profiling(True)
    try:
        _clear(outs, douts)
        R.render_device(srcs, outs, direct_outs=douts)
        pairs_dev = R.get_profile()[2]
        _same(ref, _outputs(outs, douts))
        _clear(outs, douts)
        plan.run()
        pairs_plan = R.get_profile()[2]
        _same(ref, _outputs(outs, douts))
    finally:
        R.set_profiling(False)
    assert pairs_dev == pairs_plan >= 3              # several chunks
    plan.close()
