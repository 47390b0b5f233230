"""The render kernels (k_prepare, k_render_fast, k_render<0,0>, k_render<1,0>) sample by sample against the float64
reference of tests/render_reference.py: every stem is checked on its own with check_render (local |y - y64| / scale and
global relative RMS, the bounds calibrated on the CPU emulation), never only by bit identity with another GPU render.
Each group of cases names the kernel variant it is built to reach (chunk_enqueue / arrange_chunks: one transform per
item -> k_render_fast, a long RIR in the chunk -> k_render<1,0>, everything else -> k_render<0,0>);
test_cases_reach_their_kernels confirms the mapping from the CUDA kernel names torch.profiler records."""
import ctypes
import os

import numpy as np
import pytest
import torch

import render_reference as rr
from chunk_budget import chunk_budget  # noqa: F401  (fixture)
from direct_path import direct_path_rirs, normalized
from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL

pytestmark = pytest.mark.gpu

FAST, GEN, LONG = "k_render_fast", "k_render<0,0>", "k_render<1,0>"
WORST = {}                  # kernel -> [worst local ratio, worst global relative RMS]


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    for k, (loc, glob) in sorted(WORST.items()):
        print("\nWORST %s: local %.3g, global %.3g (TAU_LOCAL %.3g, TAU_GLOBAL %.3g)" % (k, loc, glob, TAU_LOCAL, TAU_GLOBAL))


def R():
    from sonicsim_b200 import render
    return render.default_renderer()


def check(kernel, y, x, h, mode, bounds=None, idx=None, w=None, window=None, label=""):
    """One stem against render_f64 with check_render; records the worst ratios per kernel variant."""
    y = y.cpu().numpy() if isinstance(y, torch.Tensor) else np.asarray(y)
    y64, scale = rr.render_check_inputs(x, h, mode, bounds=bounds, idx=idx, w=w, window=window)
    n0 = 0 if window is None else window[0]
    r = rr.check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=n0, label="%s %s" % (kernel, label))
    cur = WORST.setdefault(kernel, [0.0, 0.0])
    cur[0], cur[1] = max(cur[0], r[0]), max(cur[1], r[1])
    return r


def plan_of(x, h, bounds):
    """(aligned, blocks) the library plans for a compact-trajectory source (ss_debug_plan)."""
    from sonicsim_b200 import _lib
    lib = _lib.load()
    P, C, L = h.shape
    s = _lib.SsSource(N=x.size, P=P, C=C, L=L, mode=_lib.SS_MOVING_BOUNDS, bounds_host=bounds.ctypes.data)
    out = np.zeros((x.size // 4096 + P + 2) * 4, np.int32)
    al = ctypes.c_int32()
    n = lib.ss_debug_plan(ctypes.byref(s), out.ctypes.data, out.size // 4, ctypes.byref(al))
    assert n >= 0
    return al.value == 1, out[:4 * n].reshape(-1, 4)


def moving(x, h, bounds, **kw):
    from sonicsim_b200 import render
    return render.MovingSource(x, h, bounds, **kw)


def host(*srcs, direct_outs=None):
    return R().render_host(list(srcs), direct_outs=direct_outs)


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def dev_source(s):
    """The device-resident twin of a host MovingSource / StaticSource (bounds_host kept)."""
    from sonicsim_b200 import render
    if isinstance(s, render.StaticSource):
        return render.StaticSource(cuda(s.dry), cuda(s.rir), s.normalize_rirs, s.direct_taps, s.window)
    return render.MovingSource(cuda(s.dry), cuda(s.rirs), cuda(s.bounds), s.bounds_host, s.normalize_rirs,
                               s.direct_taps, s.window)


def aligned_bounds(N, P, rng):
    """A trajectory for P positions over N samples whose inner waypoints sit at one common offset inside the 4096-grid
    (distinct blocks where N allows): every grid block that holds a waypoint would take two transforms, so the host cost
    rule picks aligned blocking.  With fewer blocks than waypoints, or short segments, the grid wins."""
    nb = max(1, (N - 1) // 4096)
    k = np.sort(rng.choice(np.arange(nb), P - 2, replace=nb < P - 2))
    off = int(rng.integers(1, 4096))
    cut = np.minimum(k * 4096 + off, N)
    return np.concatenate([[0], cut, [N]]).astype(np.int32)


def grid_bounds(N, P, rng):
    """Waypoints at random samples, many of them per block: the host cost rule picks the 4096-grid."""
    cut = np.sort(rng.choice(np.arange(1, N), P - 2, replace=False))
    return np.concatenate([[0], cut, [N]]).astype(np.int32)


# --------------------------------------------------------------------------------------------------- k_render_fast
@pytest.mark.parametrize("dry", ["white", "graded", "impulse"])
@pytest.mark.parametrize("rirs", ["synth", "delay"])
def test_fast_aligned_moving(dry, rirs):
    rng = np.random.default_rng(sum(map(ord, dry + rirs)))
    N, P, C, L = 70001, 7, 3, 4096
    x, h = rr.dry_signal(dry, rng, N), rr.rir_set(rirs, rng, P, C, L)
    b = rr.bounds_from_lengths([4095, 1, 8193, 4096, 4097, N - 20482])
    assert plan_of(x, h, b)[0]
    check(FAST, host(moving(x, h, b))[0], x, h, 1, bounds=b, label="aligned %s %s" % (dry, rirs))


@pytest.mark.parametrize("C", [1, 2, 3, 5])
@pytest.mark.parametrize("L", [1, 2, 4095, 4096])
def test_fast_static(C, L):
    from sonicsim_b200 import render
    rng = np.random.default_rng(C * 10000 + L)
    N = 20000
    x = rr.graded_dry(rng, N)
    h = (rr.delay_rirs(rng, 1, C, L)[0] if L % 2 else so.synth_rirs(rng, 1, C, L))[0]
    check(FAST, host(render.StaticSource(x, h))[0], x, h, 0, label="static C=%d L=%d" % (C, L))


@pytest.mark.parametrize("normalize", [False, True])
def test_fast_direct_target_and_normalize(normalize):
    rng = np.random.default_rng(77 + normalize)
    N, P, C, L, taps = 50000, 5, 2, 3000, 40
    x, h = rr.graded_dry(rng, N), (so.synth_rirs(rng, P, C, L) * 3.0).astype(np.float32)
    b = aligned_bounds(N, P, rng)
    assert plan_of(x, h, b)[0]
    hn = normalized(h) if normalize else h
    d = [np.empty((C, N), np.float32)]
    y = host(moving(x, h, b, normalize_rirs=normalize, direct_taps=taps), direct_outs=d)[0]
    check(FAST, y, x, hn, 1, bounds=b, label="reverberant normalize=%s" % normalize)
    check(FAST, d[0], x, direct_path_rirs(hn, taps), 1, bounds=b, label="direct normalize=%s" % normalize)


# --------------------------------------------------------------------------------------------------- k_render<0,0>
def test_generic_grid_from_host_cost_rule():
    rng = np.random.default_rng(5)
    N, P, C, L = 40000, 40, 3, 2000
    x, h = rr.graded_dry(rng, N), so.synth_rirs(rng, P, C, L)
    b = grid_bounds(N, P, rng)                           # ~1000-sample segments: the grid is cheaper
    assert not plan_of(x, h, b)[0]
    check(GEN, host(moving(x, h, b))[0], x, h, 1, bounds=b, label="grid bounds")


@pytest.mark.parametrize("rirs", ["synth", "delay"])
def test_generic_indexed(rirs):
    """setup_dynamic_interp's (idx, w), and non-monotone idx whose blocks span 3 to P positions (several transforms per
    block, the second and later accumulated with red_add)."""
    from sonicsim_b200 import SonicSim_moving as sm
    rng = np.random.default_rng(6)
    N, P, C, L = 30000, 9, 2, 4096
    x, h = rr.graded_dry(rng, N), rr.rir_set(rirs, rng, P, C, L)
    np.random.seed(6)
    idx, w = so.setup_dynamic_interp(so.synth_path(rng, P), N)
    check(GEN, sm.convolve_moving_receiver(x, h, idx, w), x, h, 2, idx=idx, w=w, label="setup_dynamic_interp")
    span = np.repeat(np.arange(3, 3 + (N + 4095) // 4096), 4096)[:N]            # block b spans 3 + b positions (<= P)
    span = np.minimum(span, P - 1)
    idx2 = (rng.integers(0, 1 << 20, N) % span).astype(np.int64)
    idx2[::4096] = span[::4096] - 1
    w2 = rng.random(N).astype(np.float32)
    check(GEN, sm.convolve_moving_receiver(x, h, idx2, w2), x, h, 2, idx=idx2, w=w2, label="non-monotone")


@pytest.mark.parametrize("P,kernel", [(10, FAST), (20, GEN)])
def test_device_bounds_without_host_copy(P, kernel):
    """k_blocks builds the table on the device; without bounds_host the plan is aligned iff (P - 1) 4096 <= N."""
    rng = np.random.default_rng(P)
    N, C, L = 50000, 3, 3000
    x, h = rr.graded_dry(rng, N), so.synth_rirs(rng, P, C, L)
    b = aligned_bounds(N, P, rng)
    out = torch.empty((C, N), device="cuda")
    R().render_device([moving(cuda(x), cuda(h), cuda(b))], [out])
    torch.cuda.synchronize()
    check(kernel, out, x, h, 1, bounds=b, label="device bounds P=%d" % P)


def test_generic_without_fast_kernel():
    """An aligned source in a context created with SS_NO_FAST renders with k_render<0,0>."""
    from sonicsim_b200 import _lib, render
    lib = _lib.load()
    rng = np.random.default_rng(9)
    N, P, C, L = 50000, 5, 3, 4096
    x, h = rr.graded_dry(rng, N), so.synth_rirs(rng, P, C, L)
    b = aligned_bounds(N, P, rng)
    old = os.environ.get("SS_NO_FAST")
    os.environ["SS_NO_FAST"] = "1"
    ctx = ctypes.c_void_p()
    try:
        _lib.check(lib.ss_create(_lib.default_device(), ctypes.byref(ctx)))
    finally:
        if old is None:
            del os.environ["SS_NO_FAST"]
    try:
        Rn = render.Renderer.__new__(render.Renderer)
        Rn.lib, Rn.device, Rn.ctx = lib, _lib.default_device(), ctx
        y = Rn.render_host([moving(x, h, b)])[0]
    finally:
        lib.ss_destroy(ctx)
    check(GEN, y, x, h, 1, bounds=b, label="SS_NO_FAST")


def test_host_chunk_mixing_aligned_and_grid():
    rng = np.random.default_rng(10)
    x1, h1 = rr.graded_dry(rng, 40000), so.synth_rirs(rng, 4, 2, 4096)
    b1 = aligned_bounds(40000, 4, rng)
    x2, h2 = so.synth_dry(rng, 30000), so.synth_rirs(rng, 30, 2, 500)
    b2 = grid_bounds(30000, 30, rng)
    assert plan_of(x1, h1, b1)[0] and not plan_of(x2, h2, b2)[0]
    y1, y2 = host(moving(x1, h1, b1), moving(x2, h2, b2))
    check(GEN, y1, x1, h1, 1, bounds=b1, label="aligned in a grid chunk")
    check(GEN, y2, x2, h2, 1, bounds=b2, label="grid")


# --------------------------------------------------------------------------------------------------- k_render<1,0>
@pytest.mark.parametrize("L", [4097, 8192, 8193, 9000, 32768])
def test_long_rirs(L):
    from sonicsim_b200 import render
    rng = np.random.default_rng(L)
    N, P, C = 45000, 4, 2
    x = rr.graded_dry(rng, N)
    h = rr.delay_rirs(rng, P, C, L)[0] if L % 2 else so.synth_rirs(rng, P, C, L, t60=1.0)
    b = aligned_bounds(N, P, rng)
    check(LONG, host(moving(x, h, b))[0], x, h, 1, bounds=b, label="moving L=%d" % L)
    hs = rr.rir_set("delay" if L % 2 == 0 else "synth", rng, 1, 3, L)[0]        # static, odd C
    check(LONG, host(render.StaticSource(x, hs))[0], x, hs, 0, label="static C=3 L=%d" % L)


def test_host_chunk_short_aligned_with_long():
    """DESIGN section 2: a chunk that mixes kinds renders with the most general variant present, which may round
    differently from k_render_fast; it must still meet the float64 bound."""
    rng = np.random.default_rng(12)
    x1, h1 = rr.graded_dry(rng, 40000), so.synth_rirs(rng, 5, 3, 4096)
    b1 = aligned_bounds(40000, 5, rng)
    x2, h2 = so.synth_dry(rng, 30000), so.synth_rirs(rng, 3, 2, 9000)
    b2 = aligned_bounds(30000, 3, rng)
    y1, y2 = host(moving(x1, h1, b1), moving(x2, h2, b2))
    check(LONG, y1, x1, h1, 1, bounds=b1, label="short aligned in a long chunk")
    check(LONG, y2, x2, h2, 1, bounds=b2, label="long")


# --------------------------------------------------------------------------------------------------- shape edges
@pytest.mark.parametrize("N", [1, 7, 4095, 4096, 4097, 8192, 8193, 12289])
def test_shape_edges(N):
    """P = 2, L in {1, 2, 4095, 4096, 4097} (N < L included), static and moving."""
    from sonicsim_b200 import render
    for L in (1, 2, 4095, 4096, 4097):
        rng = np.random.default_rng(N * 13 + L)
        x = rr.graded_dry(rng, N) if N > 4096 else so.synth_dry(rng, N)
        h = rr.delay_rirs(rng, 2, 3, L)[0] if L % 2 else so.synth_rirs(rng, 2, 3, L)
        b = np.array([0, N], np.int32)
        kernel = LONG if L > 4096 else FAST
        check(kernel, host(moving(x, h, b))[0], x, h, 1, bounds=b, label="P=2 N=%d L=%d" % (N, L))
        check(kernel, host(render.StaticSource(x, h[0]))[0], x, h[0], 0, label="static N=%d L=%d" % (N, L))


@pytest.mark.parametrize("L", [300, 4096, 5000])
def test_segment_edges(L):
    """Segments of 1, 4095, 4096, 4097, 8192, 8193 samples, empty segments at the start, in the middle and at the end."""
    rng = np.random.default_rng(L + 1)
    segs = [0, 1, 0, 4095, 4096, 4097, 0, 8192, 8193, 0]
    b = rr.bounds_from_lengths(segs)
    x, h = rr.graded_dry(rng, int(b[-1])), so.synth_rirs(rng, len(b), 2, L)
    kernel = LONG if L > 4096 else (FAST if plan_of(x, h, b)[0] else GEN)
    check(kernel, host(moving(x, h, b))[0], x, h, 1, bounds=b, label="segments L=%d" % L)


# --------------------------------------------------------------------------------------------------- paths
def path_batch(rng):
    """(host sources, kernel per source): aligned, static and long sources of several sizes."""
    from sonicsim_b200 import render
    srcs, kern = [], []
    for i in range(9):
        N, C = int(rng.integers(5000, 60000)), int(rng.integers(1, 6))
        x = rr.graded_dry(rng, N)
        if i % 3 == 0:
            srcs.append(render.StaticSource(x, so.synth_rirs(rng, 1, C, int(rng.integers(1, 4097)))[0]))
            kern.append(FAST)
        else:
            P = int(rng.integers(2, 6))
            L = int(rng.integers(1, 4097)) if i % 3 == 1 else int(rng.integers(4097, 12000))
            h = so.synth_rirs(rng, P, C, L)
            b = aligned_bounds(N, P, rng) if N > 4096 * P else rr.bounds_from_lengths([N] + [0] * (P - 2))
            srcs.append(moving(x, h, b, bounds_host=b))
            kern.append(kernel_of(srcs[-1]))
    return srcs, kern


def channels(s):
    from sonicsim_b200 import render
    return s.rir.shape[0] if isinstance(s, render.StaticSource) else s.rirs.shape[1]


def kernel_of(s):
    """The variant a source renders with in a chunk of its own kind (arrange_chunks)."""
    from sonicsim_b200 import render
    L = s.rir.shape[-1] if isinstance(s, render.StaticSource) else s.rirs.shape[-1]
    if L > 4096:
        return LONG
    if isinstance(s, render.StaticSource):
        return FAST
    return FAST if plan_of(s.dry, s.rirs, s.bounds)[0] else GEN


def check_source(kernel, s, y, label):
    from sonicsim_b200 import render
    if isinstance(s, render.StaticSource):
        check(kernel, y, s.dry, s.rir, 0, label=label)
    else:
        check(kernel, y, s.dry, s.rirs, 1, bounds=s.bounds, label=label)


def test_paths_device_plan_and_small_chunks(chunk_budget):
    """render_device, a plan_device run twice with the outputs NaN-filled in between, and a small chunk budget (many
    chunks over the three internal streams): every stem against float64."""
    rng = np.random.default_rng(21)
    srcs, kern = path_batch(rng)
    dev = [dev_source(s) for s in srcs]
    outs = [torch.empty((channels(s), s.dry.shape[0]), device="cuda") for s in srcs]
    R().render_device(dev, outs)
    torch.cuda.synchronize()
    for s, k, o in zip(srcs, kern, outs):
        check_source(k, s, o, "render_device")
    Rb = chunk_budget(4 << 20)
    plan = Rb.plan_device(dev, outs)
    for run in range(2):
        for o in outs:
            o.fill_(float("nan"))
        plan.run()
        torch.cuda.synchronize()
        for s, k, o in zip(srcs, kern, outs):
            check_source(k, s, o, "plan_device run %d" % run)
    plan.close()


def test_thirty_sources_global_prepare_table():
    """30 sources in one chunk: more than kPrepInline = 24, so k_prepare<false> reads the source table from memory."""
    rng = np.random.default_rng(30)
    srcs = []
    for i in range(30):
        N, P, C = int(rng.integers(9000, 20000)), int(rng.integers(2, 4)), int(rng.integers(1, 4))
        x, h = rr.graded_dry(rng, N), so.synth_rirs(rng, P, C, int(rng.integers(1, 4097)))
        srcs.append(moving(x, h, aligned_bounds(N, P, rng)))
    dev = [dev_source(s)._replace(bounds_host=s.bounds) for s in srcs]
    outs = [torch.empty((s.rirs.shape[1], s.dry.shape[0]), device="cuda") for s in srcs]
    R().render_device(dev, outs)
    torch.cuda.synchronize()
    for s, o in zip(srcs, outs):
        check_source(kernel_of(s), s, o, "30-source batch")


def test_full_size_configs1_windows():
    """A configs[1] speaker (P = 40, C = 6, L = 4096, 30 s), checked through the float64 window trick at the start, a
    waypoint, a 4096 boundary and the end."""
    rng = np.random.default_rng(2000)
    P, C, L, N = 40, 6, 4096, 480000
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
    np.random.seed(2000)
    idx, _ = so.setup_dynamic_interp(pos, N)
    b = rr.bounds_from_lengths(np.bincount(idx, minlength=P - 1))
    assert plan_of(x, h, b)[0]
    y = host(moving(x, h, b))[0]
    wp = int(b[17])
    for a, n in ((0, 6000), (wp - 3000, 6000), (4096 * 60 - 2048, 4096), (N - 6000, 6000)):
        check(FAST, y[:, a:a + n], x, h, 1, bounds=b, window=(a, n), label="configs[1] window %d" % a)


def test_cases_reach_their_kernels():
    """The kernel each group is built to reach is the one that runs (CUDA kernel names from torch.profiler)."""
    rng = np.random.default_rng(1)
    x = so.synth_dry(rng, 50000)
    ha, hl = so.synth_rirs(rng, 5, 2, 4096), so.synth_rirs(rng, 3, 2, 9000)
    b5, b3 = aligned_bounds(50000, 5, rng), aligned_bounds(50000, 3, rng)
    hg = so.synth_rirs(rng, 40, 2, 1000)
    bg = grid_bounds(50000, 40, rng)
    cases = {FAST: [moving(x, ha, b5)], LONG: [moving(x, hl, b3)], GEN: [moving(x, hg, bg)]}
    names = {FAST: "k_render_fast", GEN: "k_render<false, false>", LONG: "k_render<true, false>"}
    for k, srcs in cases.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            host(*srcs)
            torch.cuda.synchronize()
        ran = {e.name for e in prof.events() if "k_render" in e.name}
        assert any(names[k] in n for n in ran) and not any(names[o] in n for o in names if o != k for n in ran), (k, ran)
