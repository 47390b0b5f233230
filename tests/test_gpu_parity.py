"""Parity of the CUDA path (through the C ABI / drop-in functions) with the oracle and the
reference's golden vectors.  Tolerance: relative RMS <= 1e-4 per output tensor (BASELINE north star)."""
import numpy as np
import pytest
import torch

from chunk_budget import chunk_budget  # noqa: F401  (fixture)
from conftest import TOL
from oracle import sonicsim_oracle as so

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def sm():
    from sonicsim_b200 import SonicSim_moving
    return SonicSim_moving


def bounds_of(idx, P):
    return np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)


def test_native_library_is_the_code_that_runs(sm):
    sm.convolve_fixed_receiver(np.ones((1, 64), np.float32), np.ones((1, 4), np.float32))
    maps = open("/proc/self/maps").read()
    assert "libsonicsim_b200.so" in maps


def test_golden_fixed(sm, golden):
    g = golden("convolve_fixed_receiver")
    for k in range(int(g["n_cases"])):
        y = sm.convolve_fixed_receiver(g[f"x{k}"], g[f"h{k}"])
        assert isinstance(y, np.ndarray) and y.dtype == np.float32 and y.shape == g[f"y{k}"].shape
        assert so.rel_rms(y, g[f"y{k}"]) < TOL
        y_t = sm.convolve_fixed_receiver(torch.from_numpy(g[f"x{k}"]), torch.from_numpy(g[f"h{k}"]))   # SonicSet.py:93
        assert np.array_equal(y, y_t)


def test_golden_moving(sm, golden):
    g = golden("convolve_moving_receiver")
    for k in range(int(g["n_cases"])):
        y = sm.convolve_moving_receiver(g[f"x{k}"], g[f"h{k}"], g[f"idx{k}"].astype(np.int64), g[f"w{k}"])
        assert y.dtype == np.float32 and y.shape == g[f"y{k}"].shape
        assert so.rel_rms(y, g[f"y{k}"]) < TOL


def test_golden_interpolate_moving_audio(sm, golden):
    g = golden("interpolate_moving_audio")
    for k in range(int(g["n_cases"])):
        np.random.seed(int(g[f"seed{k}"]))
        y = sm.interpolate_moving_audio(torch.from_numpy(g[f"x{k}"]), torch.from_numpy(g[f"h{k}"]),
                                        [list(p) for p in g[f"pos{k}"]])
        assert isinstance(y, torch.Tensor) and y.dtype == torch.float32 and not y.is_cuda
        assert so.rel_rms(y.numpy(), g[f"y{k}"]) < TOL
        # list-of-tensors form of ir1_list (SonicSim_moving.py:122 np.array(list))
        np.random.seed(int(g[f"seed{k}"]))
        y2 = sm.interpolate_moving_audio(torch.from_numpy(g[f"x{k}"]), [torch.from_numpy(t) for t in g[f"h{k}"]],
                                         g[f"pos{k}"])
        assert np.array_equal(y.numpy(), y2.numpy())


@pytest.mark.parametrize("P,C,L,N", [(3, 1, 1, 100), (2, 2, 4096, 4096), (2, 1, 4097, 8193), (9, 3, 600, 12289),
                                     (5, 2, 9000, 5000), (40, 6, 4096, 100000), (13, 5, 257, 70001),
                                     (200, 2, 300, 50000)])          # many short segments: the grid plan is chosen
def test_shapes_and_partitions(sm, P, C, L, N):
    rng = np.random.default_rng(P * 1000 + L)
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
    np.random.seed(7)
    idx, w = so.setup_dynamic_interp(pos, N)
    ref = so.convolve_moving_receiver(x, h, idx, w)
    assert so.rel_rms(sm.convolve_moving_receiver(x, h, idx, w), ref) < TOL
    # compact-trajectory form of the same render (aligned or grid blocking, whichever is cheaper)
    from sonicsim_b200 import render
    bounds = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)
    y = render.default_renderer().render_host([render.MovingSource(x, h, bounds)])[0]
    assert so.rel_rms(y, ref) < TOL


def test_empty_segments_ragged_and_random_indices(sm):
    rng = np.random.default_rng(3)
    P, C, L, N = 9, 2, 40, 5
    x, pos = so.synth_dry(rng, N), so.synth_path(rng, P)
    h = rng.standard_normal((P, C, L)).astype(np.float32)
    pos[3] = pos[2]
    for seed in range(50):
        np.random.seed(seed)
        try:
            idx, w = so.setup_dynamic_interp(pos, N)
            break
        except ValueError:
            continue
    assert so.rel_rms(sm.convolve_moving_receiver(x, h, idx, w), so.convolve_moving_receiver(x, h, idx, w)) < TOL
    # arbitrary (non-monotone) index / weight arrays
    P, C, L, N = 7, 2, 300, 9000
    x, h = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L)
    idx = rng.integers(0, P - 1, N)
    w = rng.random(N).astype(np.float32)
    assert so.rel_rms(sm.convolve_moving_receiver(x, h, idx, w), so.convolve_moving_receiver(x, h, idx, w)) < TOL
    with pytest.raises(IndexError):
        sm.convolve_moving_receiver(x, h, np.full(N, P - 1), w)


def test_batch_api_matches_single_calls_and_device_path(sm):
    from sonicsim_b200 import render
    rng = np.random.default_rng(11)
    moving, static = [], []
    for i in range(5):
        N = 20000 + 3000 * i
        P = 4 + i
        moving.append((so.synth_dry(rng, N), so.synth_rirs(rng, P, 3, 700 + 100 * i), so.synth_path(rng, P)))
    for i in range(3):
        static.append((so.synth_dry(rng, 15000), so.synth_rirs(rng, 1, 2 + i, 512)[0]))
    np.random.seed(5)
    ym, ys = render.render_scene(moving, static)
    np.random.seed(5)
    for (x, h, pos), y in zip(moving, ym):
        idx, w = so.setup_dynamic_interp(pos, x.shape[0])
        assert so.rel_rms(y, so.convolve_moving_receiver(x, h, idx, w)) < TOL
    for (x, h), y in zip(static, ys):
        assert so.rel_rms(y, so.convolve_fixed_receiver(x[None], h)) < TOL
    # device-resident path gives bit-identical results to the host path
    R = render.default_renderer()
    np.random.seed(5)
    srcs, outs = [], []
    for (x, h, pos) in moving:
        b = render.trajectory_bounds(pos, x.shape[0])
        srcs.append(render.MovingSource(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), torch.from_numpy(b).cuda()))
        outs.append(torch.empty((h.shape[1], x.shape[0]), device="cuda"))
    R.render_device(srcs, outs)
    torch.cuda.synchronize()
    for y, o in zip(ym, outs):
        assert np.array_equal(y, o.cpu().numpy())


def test_full_size_cfg2_against_oracle_and_properties(sm):
    """BASELINE configs[1] shape: C=6, P=40, L=4096, N=480000 (one speaker)."""
    rng = np.random.default_rng(2000)
    P, C, L, N = 40, 6, 4096, 480000
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
    np.random.seed(2000)
    idx, w = so.setup_dynamic_interp(pos, N)
    y = sm.convolve_moving_receiver(x, h, idx, w)
    ref = so.convolve_moving_receiver(x, h, idx, w)
    assert so.rel_rms(y, ref) < TOL
    # compact-trajectory path (interpolate_moving_audio): same weights computed on the device
    np.random.seed(2000)
    y2 = sm.interpolate_moving_audio(torch.from_numpy(x[None]), torch.from_numpy(h[:, None]), pos).numpy()
    print("idx-vs-bounds path: rel-RMS %.3g, max abs diff %.3g" % (so.rel_rms(y2, y), np.abs(y2 - y).max()))
    assert so.rel_rms(y2, y) < 2e-6            # waypoint-aligned blocks (bounds) vs grid blocks (idx, w)
    # linearity in the RIR set
    h2 = so.synth_rirs(rng, P, C, L)
    ya = sm.convolve_moving_receiver(x, h2, idx, w)
    yab = sm.convolve_moving_receiver(x, (h + 0.5 * h2).astype(np.float32), idx, w)
    assert so.rel_rms(yab, y + 0.5 * ya) < 1e-5
    # delta RIR -> identity; boundary continuity of the interpolation
    hd = np.zeros((P, C, L), np.float32)
    hd[:, :, 0] = 1.0
    yd = sm.convolve_moving_receiver(x, hd, idx, w)
    assert so.rel_rms(yd, np.broadcast_to(x, (C, N))) < 2e-6


def test_long_rir_partitioned_cfg4_shape_reduced(sm):
    """configs[3] flavour: L = 32768 (8 partitions), 4 channels; N reduced so the oracle runs in seconds."""
    rng = np.random.default_rng(4000)
    P, C, L, N = 12, 4, 32768, 200000
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L, sr=48000, t60=1.5), so.synth_path(rng, P)
    np.random.seed(4000)
    idx, w = so.setup_dynamic_interp(pos, N)
    assert so.rel_rms(sm.convolve_moving_receiver(x, h, idx, w), so.convolve_moving_receiver(x, h, idx, w)) < TOL
    assert so.rel_rms(sm.convolve_fixed_receiver(x[None], h[0]), so.convolve_fixed_receiver(x[None], h[0])) < TOL


def test_large_mixed_batch_multi_chunk_two_streams(chunk_budget):
    """Many heterogeneous sources in one device-path call (several chunks, alternating streams, both
    blocking modes, long RIRs, static sources) == the same sources rendered one by one."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(99)
    R = chunk_budget(8 << 20)                       # force many chunks
    srcs_np = []
    for i in range(23):
        N = int(rng.integers(3000, 90000))
        C = int(rng.integers(1, 7))
        kind = i % 4
        if kind == 0:
            srcs_np.append(("static", so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, int(rng.integers(8, 3000)))[0]))
        else:
            P = int(rng.integers(2, 12))
            L = int(rng.integers(8, 3000)) if kind != 3 else int(rng.integers(4097, 9000))
            pos = so.synth_path(rng, P)
            np.random.seed(i)
            srcs_np.append(("moving", so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), render.trajectory_bounds(pos, N)))
    dev, outs = [], []
    for s in srcs_np:
        if s[0] == "static":
            dev.append(render.StaticSource(torch.from_numpy(s[1]).cuda(), torch.from_numpy(s[2]).cuda()))
            outs.append(torch.empty((s[2].shape[0], s[1].shape[0]), device="cuda"))
        else:
            bh = s[3] if len(dev) % 2 == 0 else None          # mix host-built and device-built block tables
            dev.append(render.MovingSource(torch.from_numpy(s[1]).cuda(), torch.from_numpy(s[2]).cuda(),
                                           torch.from_numpy(s[3]).cuda(), bh))
            outs.append(torch.empty((s[2].shape[1], s[1].shape[0]), device="cuda"))
    R.render_device(dev, outs)
    torch.cuda.synchronize()
    for s, o, dsrc in zip(srcs_np, outs, dev):
        if s[0] == "static":
            one = R.render_host([render.StaticSource(s[1], s[2])])[0]
            ref = so.convolve_fixed_receiver(s[1][None], s[2])
        else:
            one = R.render_host([render.MovingSource(s[1], s[2], s[3])])[0]
            idx = np.repeat(np.arange(len(s[3]) - 1), np.diff(s[3]))
            w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(s[3])]).astype(np.float32)
            ref = so.convolve_moving_receiver(s[1], s[2], idx, w)
        same_plan = s[0] == "static" or dsrc.bounds_host is not None      # without host bounds the blocking plan is a heuristic
        if same_plan:
            assert np.array_equal(o.cpu().numpy(), one)
        else:
            assert so.rel_rms(o.cpu().numpy(), one) < 2e-6
        assert so.rel_rms(one, ref) < TOL


def test_many_small_sources_in_one_chunk():
    """More sources in one chunk than k_prepare takes as kernel parameters (24): the global-table variant of the
    kernel == the same sources rendered one by one (parameter variant)."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(7)
    R = render.default_renderer()
    srcs, dev, outs = [], [], []
    for i in range(41):
        N, C, P, L = int(rng.integers(2000, 9000)), int(rng.integers(1, 4)), int(rng.integers(2, 6)), int(rng.integers(8, 700))
        x, h = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L)
        np.random.seed(100 + i)
        b = render.trajectory_bounds(so.synth_path(rng, P), N)
        srcs.append((x, h, b))
        dev.append(render.MovingSource(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), torch.from_numpy(b).cuda(), b))
        outs.append(torch.empty((C, N), device="cuda"))
    plan = R.plan_device(dev, outs)                  # bound once, run twice (second run after the outputs were cleared)
    plan.run()
    torch.cuda.synchronize()
    first = [o.clone() for o in outs]
    for o in outs:
        o.zero_()
    plan.run()
    torch.cuda.synchronize()
    for (x, h, b), o, f in zip(srcs, outs, first):
        one = R.render_host([render.MovingSource(x, h, b)])[0]
        assert np.array_equal(o.cpu().numpy(), one) and torch.equal(o, f)
    x, h, b = srcs[0]
    idx = np.repeat(np.arange(len(b) - 1), np.diff(b))
    w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(b)]).astype(np.float32)
    assert so.rel_rms(outs[0].cpu().numpy(), so.convolve_moving_receiver(x, h, idx, w)) < TOL


def test_host_plan_rerun_with_refilled_buffers():
    """Renderer.plan_host binds buffers once; run() picks up new buffer contents (and new trajectories) each time."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(123)
    N, C, L, P = 30000, 2, 900, 5
    x = so.synth_dry(rng, N)
    h = so.synth_rirs(rng, P, C, L)
    np.random.seed(1)
    bounds = render.trajectory_bounds(so.synth_path(rng, P), N)
    xs, hs_ = so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, L)[0]
    R = render.default_renderer()
    plan = R.plan_host([render.MovingSource(x, h, bounds), render.StaticSource(xs, hs_)], lufs_targets=[-20.0, None])
    for it in range(3):
        outs = plan.run()
        idx = np.repeat(np.arange(P - 1), np.diff(bounds))
        w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(bounds)]).astype(np.float32)
        ref = so.lufs_norm(np.ascontiguousarray(so.convolve_moving_receiver(x, h, idx, w).T), 16000, -20.0)[0].T
        assert so.rel_rms(outs[0], ref) < TOL
        assert so.rel_rms(outs[1], so.convolve_fixed_receiver(xs[None], hs_)) < TOL
        lufs, gain = plan.loudness()[0]
        assert np.isfinite(lufs) and gain > 0
        # refill the bound buffers in place: new dry signal, new RIRs, new trajectory
        x[:] = so.synth_dry(rng, N)
        h[:] = so.synth_rirs(rng, P, C, L)
        np.random.seed(10 + it)
        bounds[:] = render.trajectory_bounds(so.synth_path(rng, P), N)
        xs[:] = so.synth_dry(rng, N)


def test_device_plan_is_one_graph_launch_and_matches_direct_launches(chunk_budget):
    """Renderer.plan_device -> ss_plan_*: descriptors + scratch resident, launches captured into a CUDA graph (several
    chunks forked over the internal streams).  Must equal ss_render_dev bit for bit, pick up refilled buffers, and
    reject tensors that would make the kernels write out of bounds (ADVICE r1)."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(321)
    R = chunk_budget(8 << 20)                       # several chunks -> fork / join inside the graph
    dev, outs, host = [], [], []
    for i in range(9):
        N, C, P = int(rng.integers(20000, 60000)), int(rng.integers(1, 5)), int(rng.integers(2, 9))
        L = int(rng.integers(100, 4096)) if i % 3 else int(rng.integers(4097, 7000))
        x, h = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L)
        np.random.seed(40 + i)
        b = render.trajectory_bounds(so.synth_path(rng, P), N)
        host.append((x, h, b))
        dev.append(render.MovingSource(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), torch.from_numpy(b).cuda(),
                                       b if i % 2 == 0 else None))
        outs.append(torch.empty((C, N), device="cuda"))
    xs, hs_ = so.synth_dry(rng, 30000), so.synth_rirs(rng, 1, 3, 700)[0]
    dev.append(render.StaticSource(torch.from_numpy(xs).cuda(), torch.from_numpy(hs_).cuda()))
    outs.append(torch.empty((3, 30000), device="cuda"))
    direct = [torch.empty_like(o) for o in outs]
    R.render_device(dev, direct)
    plan = R.plan_device(dev, outs)
    n0 = R.launch_count()
    plan.run()
    torch.cuda.synchronize()
    assert plan.is_graph()
    assert R.launch_count() > n0                  # the graph's kernels are counted
    for o, d in zip(outs, direct):
        assert torch.equal(o, d)
    # refill one dry signal in place: the next run must see it
    x0 = so.synth_dry(rng, host[0][0].shape[0])
    dev[0].dry.copy_(torch.from_numpy(x0))
    for o in outs:
        o.zero_()
    plan.run()
    torch.cuda.synchronize()
    one = R.render_host([render.MovingSource(x0, host[0][1], host[0][2])])[0]
    assert np.array_equal(outs[0].cpu().numpy(), one)
    for o, d in zip(outs[1:], direct[1:]):
        assert torch.equal(o, d)
    plan.close()
    # validation of device tensors
    with pytest.raises(ValueError):
        R.plan_device([dev[0]], [torch.empty((outs[0].shape[0], outs[0].shape[1] - 1), device="cuda")])
    with pytest.raises(ValueError):
        R.plan_device([dev[0]], [outs[0].double()])
    with pytest.raises(ValueError):
        R.plan_device([render.MovingSource(dev[0].dry, dev[0].rirs.transpose(1, 2), dev[0].bounds)], [outs[0]])
    with pytest.raises(ValueError):
        R.plan_device([render.MovingSource(dev[0].dry.cpu(), dev[0].rirs, dev[0].bounds)], [outs[0]])


def test_device_path_reports_trajectories_it_cannot_refuse():
    """ss_render_dev takes device pointers and cannot check idx / bounds up front like the host path does (IndexError /
    ValueError there).  Kernels that meet an out-of-contract trajectory clamp, and set a flag that
    Renderer.check_device_errors turns into the reference's exception types (ADVICE r1)."""
    import ctypes
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    R.check_device_errors()                               # clean so far
    rng = np.random.default_rng(8)
    P, C, L, N = 5, 2, 300, 20000
    x, h = torch.from_numpy(so.synth_dry(rng, N)).cuda(), torch.from_numpy(so.synth_rirs(rng, P, C, L)).cuda()
    out = torch.empty((C, N), device="cuda")
    idx = torch.randint(0, P - 1, (N,), dtype=torch.int32, device="cuda")
    w = torch.rand(N, device="cuda")
    item = (_lib.SsSource * 1)(_lib.SsSource(x=x.data_ptr(), rir=h.data_ptr(), out=out.data_ptr(), idx=idx.data_ptr(), w=w.data_ptr(),
                                             N=N, P=P, C=C, L=L, mode=_lib.SS_MOVING_INDEXED))
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(R.lib.ss_render_dev(R.ctx, item, 1, stream))
    R.check_device_errors()                               # valid indices: nothing to report
    ref = so.convolve_moving_receiver(x.cpu().numpy(), h.cpu().numpy(), idx.cpu().numpy().astype(np.int64), w.cpu().numpy())
    assert so.rel_rms(out.cpu().numpy(), ref) < TOL
    idx[N // 2] = P - 1                                   # idx + 1 == P: the reference raises IndexError
    _lib.check(R.lib.ss_render_dev(R.ctx, item, 1, stream))
    with pytest.raises(IndexError):
        R.check_device_errors()
    R.check_device_errors()                               # the flag is cleared by reading it
    # device-only bounds table that does not end at N (many short segments -> grid blocking, where it is checked)
    P2 = 20
    h2 = torch.from_numpy(so.synth_rirs(rng, P2, C, L)).cuda()
    bounds = torch.linspace(0, N, P2).to(torch.int32).cuda()
    out2 = [torch.empty((C, N), device="cuda")]
    R.render_device([render.MovingSource(x, h2, bounds)], out2)
    R.check_device_errors()
    bounds[-1] = N - 5
    R.render_device([render.MovingSource(x, h2, bounds)], out2)
    with pytest.raises(ValueError):
        R.check_device_errors()


def test_fast_kernel_gives_the_same_bits_run_after_run(chunk_budget):
    """k_render_fast hands its buffers over through mbarriers, a cp.async item ring and a last-warp-out election.  A
    lost hand-over would show as a changed sample: 40 runs of a multi-chunk batch (several items per CTA, X kept and
    replaced) must all equal the first one bit for bit, and the first must match the oracle."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(2024)
    R = chunk_budget(24 << 20)
    dev, outs, host = [], [], []
    for i in range(10):
        N, P, C, L = 200000 + 4096 * i, 14, 6, 4096
        x, h = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L)
        np.random.seed(300 + i)
        b = render.trajectory_bounds(so.synth_path(rng, P), N)
        host.append((x, h, b))
        dev.append(render.MovingSource(torch.from_numpy(x).cuda(), torch.from_numpy(h).cuda(), torch.from_numpy(b).cuda(), b))
        outs.append(torch.empty((C, N), device="cuda"))
    plan = R.plan_device(dev, outs)
    plan.run()
    torch.cuda.synchronize()
    first = [o.clone() for o in outs]
    for _ in range(40):
        for o in outs:
            o.fill_(float("nan"))
        plan.run()
        torch.cuda.synchronize()
        for o, f in zip(outs, first):
            assert torch.equal(o, f)
    x, h, b = host[3]
    idx = np.repeat(np.arange(len(b) - 1), np.diff(b))
    w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(b)]).astype(np.float32)
    assert so.rel_rms(first[3].cpu().numpy(), so.convolve_moving_receiver(x, h, idx, w)) < TOL
    plan.close()
