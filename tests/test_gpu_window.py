"""Time windows through the real kernels.  Every windowed stem equals, bit for bit, the same samples of the full render
- through ss_render_host (default context and one with a 1 MB host pipeline budget), ss_render_dev with and without
bounds_host, and a device plan run twice with the dry signal changed in between, all through the C ABI - while every
input outside the documented read set is NaN (or an out-of-range position), and every output lies inside a larger
buffer with sentinels on both sides.  Also the Python API, windowed and unwindowed sources in one batch, BASELINE
configs[1] speakers against the oracle, and the argument checks."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import TOL
from oracle import sonicsim_oracle as so
from window_cases import CASES, _bad_bounds, _host_aligned, make_case, poison, read_set, windows
from gpu_plumbing import _lib, small_host_budget_context

pytestmark = pytest.mark.gpu

SENT = np.float32(1234.5)
PAD = 37


class Batch:
    """One case rendered as [full source] + [one windowed source per window], every windowed source reading its own
    copy of the inputs, poisoned outside the read set of the path (`host_visible`: the trajectory is visible on the host)
    and writing into a padded buffer with sentinels."""

    def __init__(self, name, normalize, direct, dev, host_visible, aligned, wins, x=None):
        L_, _ = _lib()
        self.name, self.mode = name, CASES[name][0]
        mode, P, C, Lr, N, taps = CASES[name]
        x0, h, idx, w, bounds, _ = make_case(name)
        self.x = x0 if x is None else x
        self.h, self.idx, self.w, self.bounds = h, idx, w, bounds
        self.C, self.N, self.dev, self.wins = C, N, dev, wins
        self.taps = taps if direct else 0
        flags = (L_.SS_RIR_NORMALIZE if normalize else 0) | (L_.SS_DIRECT_TARGET if direct else 0)
        self.keep, self.items, self.outs = [], [], []
        arr = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if dev else np.ascontiguousarray
        ptr = (lambda a: a.data_ptr()) if dev else (lambda a: a.ctypes.data)
        self.arr, self.ptr = arr, ptr
        self.inputs = []
        for k, win in enumerate([None] + list(wins)):
            if win is None:
                xs, hs, ids, ws_ = self.x, h, idx, w
            else:
                rs = read_set(mode, P, C, Lr, N, bounds, aligned, win, normalize, host_visible)
                xs, hs, ids, ws_ = poison(self.x, h, idx if mode == 2 else None, w if mode == 2 else None, rs)
            n = N if win is None else win[1]
            bufs = []
            for _ in range(2 if direct else 1):
                b = np.full(C * n + 2 * PAD, np.nan, np.float32)
                b[:PAD] = SENT
                b[-PAD:] = SENT
                bufs.append(arr(b))
            dx, dh = arr(xs), arr(hs if mode else hs)
            it = L_.SsSource(x=ptr(dx), rir=ptr(dh), N=N, P=P, C=C, L=Lr, mode=mode, flags=flags)
            it.out = ptr(bufs[0]) + 4 * PAD
            if direct:
                it.out_direct = ptr(bufs[1]) + 4 * PAD
                it.direct_taps = taps
            keep = [dx, dh, bufs]
            if mode == 1:
                db = arr(bounds)
                it.bounds = ptr(db)
                if host_visible and dev:
                    hb = np.ascontiguousarray(bounds, np.int32)
                    it.bounds_host = hb.ctypes.data
                    keep.append(hb)
                keep.append(db)
            elif mode == 2:
                di, dw = arr(ids), arr(ws_)
                it.idx, it.w = ptr(di), ptr(dw)
                keep += [di, dw]
            if win is not None:
                it.win_start, it.win_len = win
            self.items.append(it)
            self.keep.append(keep)
            self.outs.append((bufs, n))
            self.inputs.append((dx, xs))

    def array(self):
        return (self.items[0].__class__ * len(self.items))(*self.items)

    def set_x(self, x2, aligned, normalize, host_visible):
        """Overwrite every item's dry signal in place (the windowed ones poisoned as before)."""
        mode, P, C, Lr, N, _ = CASES[self.name]
        for k, win in enumerate([None] + list(self.wins)):
            xs = x2 if win is None else poison(x2, self.h, None, None, read_set(
                mode, P, C, Lr, N, self.bounds, aligned, win, normalize, host_visible))[0]
            dx = self.inputs[k][0]
            if self.dev:
                dx.copy_(torch.from_numpy(xs))
            else:
                dx[:] = xs
        self.x = x2

    def reset(self):
        for bufs, n in self.outs:
            for b in bufs:
                if self.dev:
                    b[PAD:-PAD].fill_(float("nan"))
                else:
                    b[PAD:-PAD] = np.nan

    def check(self, ref=None):
        """Windows == full[:, a:a+n] bit for bit, every in-window value written, sentinels untouched; the full stem
        equals `ref` (a render without windows) when given."""
        host = (lambda t: t.cpu().numpy()) if self.dev else (lambda t: t)
        stems = []
        for bufs, n in self.outs:
            got = []
            for b in bufs:
                a = host(b)
                assert np.all(a[:PAD] == SENT) and np.all(a[-PAD:] == SENT), self.name
                v = a[PAD:-PAD].reshape(self.C, n)
                assert not np.isnan(v).any(), self.name
                got.append(v)
            stems.append(got)
        full = stems[0]
        if ref is not None:
            for f, r in zip(full, ref):
                assert np.array_equal(f, r), self.name
        for (a, n), got in zip(self.wins, stems[1:]):
            for g, f in zip(got, full):
                assert np.array_equal(g, f[:, a:a + n]), (self.name, (a, n))
        return full


FLAGS = [(False, False), (True, False), (False, True), (True, True)]
FLAG_IDS = ["plain", "normalize", "direct", "normalize+direct"]


def _setup(name):
    mode, P, C, Lr, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    K = (Lr + 4095) // 4096
    al_host = _host_aligned(mode, P, C, Lr, N, bounds)
    al_dev = 1 if mode == 1 and K == 1 and (P - 1) * 4096 <= N else 0        # the rule without bounds_host
    wins = windows(name, N, bounds if mode == 1 else None, al_host, seed=3)
    return x, al_host, al_dev, wins


def _reference(name, normalize, direct):
    """The full stem(s) of the source without windows, alone in a call of the host path."""
    b = Batch(name, normalize, direct, False, True, 0, [])
    L_, R = _lib()
    L_.check(R.lib.ss_render_host(R.ctx, b.array(), 1))
    return b.check()


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
@pytest.mark.parametrize("name", list(CASES))
def test_window_bits_on_every_path(name, flags):
    normalize, direct = flags
    L_, R = _lib()
    x, al_host, al_dev, wins = _setup(name)
    ref = _reference(name, normalize, direct)
    # host path, default context and 1 MB pipeline chunks
    b = Batch(name, normalize, direct, False, True, al_host, wins)
    L_.check(R.lib.ss_render_host(R.ctx, b.array(), len(b.items)))
    b.check(ref)
    with small_host_budget_context() as ctx:
        b.reset()
        L_.check(R.lib.ss_render_host(ctx, b.array(), len(b.items)))
        b.check(ref)
    # device path with and without bounds_host
    for visible, al in ((True, al_host), (False, al_dev)):
        b = Batch(name, normalize, direct, True, visible, al, wins)
        L_.check(R.lib.ss_render_dev(R.ctx, b.array(), len(b.items), None))
        torch.cuda.synchronize()
        full = b.check(ref if al == al_host else None)
        bits = ctypes.c_uint32()
        L_.check(R.lib.ss_device_errors(R.ctx, ctypes.byref(bits)))
        assert bits.value == 0
    # a plan, run twice with x changed in between (bounds_host: the trajectory is visible on the host)
    b = Batch(name, normalize, direct, True, True, al_host, wins)
    items = b.array()
    plan = ctypes.c_void_p()
    L_.check(R.lib.ss_plan_create(R.ctx, items, len(b.items), ctypes.byref(plan)))
    try:
        fulls = []
        for k in range(2):
            if k == 1:
                b.set_x(so.synth_dry(np.random.default_rng(99), b.N), al_host, normalize, True)
            b.reset()
            L_.check(R.lib.ss_plan_run(plan, None))
            torch.cuda.synchronize()
            fulls.append(b.check(ref if k == 0 else None))
        assert not np.array_equal(fulls[0][0], fulls[1][0])
    finally:
        R.lib.ss_plan_destroy(plan)


@pytest.mark.parametrize("name", ["bounds", "static2", "long"])
def test_python_api_windows(name):
    """render_host, plan_host, render_device and plan_device with (C, length) outputs."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    mode, P, C, Lr, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    wins = windows(name, N, bounds if mode == 1 else None, _host_aligned(mode, P, C, Lr, N, bounds))
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()

    def src(win, dev=False):
        t = to if dev else (lambda a: a)
        if mode == 0:
            return render.StaticSource(t(x), t(h[0]), False, taps, win)
        return render.MovingSource(t(x), t(h), t(bounds), bounds if dev else None, False, taps, win)
    full_d = np.empty((C, N), np.float32)
    full = R.render_host([src(None)], direct_outs=[full_d])[0]
    dd = [np.empty((C, n), np.float32) for _, n in wins]
    outs = R.render_host([src(win) for win in wins], direct_outs=dd)
    hp = R.plan_host([src(win) for win in wins], direct_outs=[np.empty((C, n), np.float32) for _, n in wins])
    pouts = hp.run()
    douts = [torch.empty((C, n), device="cuda") for _, n in wins]
    ddouts = [torch.empty((C, n), device="cuda") for _, n in wins]
    R.render_device([src(win, True) for win in wins], douts, direct_outs=ddouts)
    pl = R.plan_device([src(win, True) for win in wins], [torch.empty((C, n), device="cuda") for _, n in wins],
                       direct_outs=[torch.empty((C, n), device="cuda") for _, n in wins])
    pl.run()
    torch.cuda.synchronize()
    for k, (a, n) in enumerate(wins):
        for got in (outs[k], pouts[k], douts[k].cpu().numpy(), pl._keep[1][k].cpu().numpy()):
            assert np.array_equal(got, full[:, a:a + n]), (name, a, n)
        for got in (dd[k], ddouts[k].cpu().numpy(), pl._keep[2][k].cpu().numpy()):
            assert np.array_equal(got, full_d[:, a:a + n]), (name, a, n)


def test_mixed_batch_keeps_unwindowed_bits():
    """Windowed and unwindowed sources in one batch: on each path the unwindowed stems keep the bits of the same batch
    without windows, and the windowed ones are its slices.  (Each path against itself: the host path may run an
    aligned source through the generic kernel, which a chunk with a long RIR needs, the device path through the fast
    one, and those two kernels need not round alike.)"""
    from sonicsim_b200 import render
    R = render.default_renderer()
    srcs, wins = [], []
    for name in ("bounds", "static2", "long", "bounds3"):
        mode, P, C, Lr, N, taps = CASES[name]
        x, h, idx, w, bounds, _ = make_case(name)
        s = render.StaticSource(x, h[0]) if mode == 0 else render.MovingSource(x, h, bounds)
        srcs.append(s)
        wins.append((N // 3, N // 4))
    windowed = lambda ss: [s if k % 2 else s._replace(window=wins[k]) for k, s in enumerate(ss)]
    plain = R.render_host(srcs)
    mixed = R.render_host(windowed(srcs))
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dsrcs = [render.StaticSource(to(s.dry), to(s.rir)) if isinstance(s, render.StaticSource)
             else render.MovingSource(to(s.dry), to(s.rirs), to(s.bounds), s.bounds) for s in srcs]
    dplain = [torch.empty(p.shape, device="cuda") for p in plain]
    R.render_device(dsrcs, dplain)
    dmixed = [torch.empty((p.shape[0], wins[k][1] if k % 2 == 0 else p.shape[1]), device="cuda")
              for k, p in enumerate(plain)]
    R.render_device(windowed(dsrcs), dmixed)
    torch.cuda.synchronize()
    for path, ref, got in (("host", plain, mixed),
                           ("device", [t.cpu().numpy() for t in dplain], [t.cpu().numpy() for t in dmixed])):
        for k, p in enumerate(ref):
            a, n = wins[k]
            assert np.array_equal(got[k], p if k % 2 else p[:, a:a + n]), (path, k)


def test_cfg2_speakers_four_second_crops_against_the_oracle():
    """BASELINE configs[1] speakers (P = 40, C = 6, L = 4096, 30 s at 16 kHz): 4 s crops against the oracle's slice."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(4242)
    N, C, L, P, sr = 480000, 6, 4096, 40, 16000
    dry, pos, h = so.synth_dry(rng, N), so.synth_path(rng, P), so.synth_rirs(rng, P, C, L)
    np.random.seed(4242)
    bounds = render.trajectory_bounds(pos, N)
    idx = np.repeat(np.arange(P - 1), np.diff(bounds))
    w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(bounds)]).astype(np.float32)
    ref = so.convolve_moving_receiver(dry, h, idx, w)
    wins = [(0, 4 * sr), (123457, 4 * sr), (N - 4 * sr, 4 * sr)]
    outs = render.default_renderer().render_host([render.MovingSource(dry, h, bounds, window=win) for win in wins])
    for (a, n), o in zip(wins, outs):
        assert so.rel_rms(o, ref[:, a:a + n]) < TOL


def test_window_errors():
    from sonicsim_b200 import render
    L_, R = _lib()
    x, h, idx, w, bounds, taps = make_case("indexed")
    P, C, Lr = h.shape
    N = x.shape[0]
    out = np.zeros((C, N), np.float32)

    def item(win):
        return L_.SsSource(x=x.ctypes.data, rir=h.ctypes.data, out=out.ctypes.data, idx=idx.ctypes.data,
                           w=w.ctypes.data, N=N, P=P, C=C, L=Lr, mode=L_.SS_MOVING_INDEXED,
                           win_start=win[0], win_len=win[1])
    for win in [(0, -1), (-1, 10), (5, 0), (N - 10, 11), (0x7fffffff, 0x7fffffff)]:
        one = (L_.SsSource * 1)(item(win))
        assert R.lib.ss_render_host(R.ctx, one, 1) == L_.SS_ERR_INVALID
        assert R.lib.ss_render_dev(R.ctx, one, 1, None) == L_.SS_ERR_INVALID
        plan = ctypes.c_void_p()
        assert R.lib.ss_plan_create(R.ctx, one, 1, ctypes.byref(plan)) == L_.SS_ERR_INVALID
    # a loudness target on a windowed source: refused before any copy
    from sonicsim_b200.SonicSim_audio import gating_plan
    brk, blo, bhi = gating_plan(N, 16000.0, 0.4)
    res = np.zeros(2)
    post = (L_.SsPostLufs * 1)(L_.SsPostLufs(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data,
                                             n_e=len(brk) - 1, n_blocks=len(blo), rate=16000.0, block_size=0.4,
                                             target_lufs=-23.0, result=res.ctypes.data))
    sentinel = np.full((C, 100), 7.0, np.float32)
    it = item((10, 100))
    it.out = sentinel.ctypes.data
    assert R.lib.ss_render_host_ex(R.ctx, (L_.SsSource * 1)(it), 1, post) == L_.SS_ERR_INVALID
    assert np.all(sentinel == 7.0)
    # a windowed source whose bounds break the contract (ascending from 0 to N) is refused before anything is planned
    Nb = 40960
    good, bad = _bad_bounds(Nb)
    Pb = len(good)
    xg, hg = np.zeros(Nb, np.float32), np.zeros((Pb, 2, 300), np.float32)
    og = np.zeros((2, 1000), np.float32)
    for b in [good] + bad:
        b32 = np.ascontiguousarray(b, np.int32)
        it = L_.SsSource(x=xg.ctypes.data, rir=hg.ctypes.data, out=og.ctypes.data, bounds=b32.ctypes.data, N=Nb, P=Pb,
                         C=2, L=300, mode=L_.SS_MOVING_BOUNDS, win_start=5000, win_len=1000)
        want = L_.SS_OK if b is good else L_.SS_ERR_INVALID
        assert R.lib.ss_render_host(R.ctx, (L_.SsSource * 1)(it), 1) == want
        if b is not good:
            with pytest.raises(ValueError):
                R.render_host([render.MovingSource(xg, hg, b32, window=(5000, 1000))])
    # the Python layer
    xb, hb, _, _, bb, tb = make_case("bounds")
    Cb, Nb = hb.shape[1], xb.shape[0]
    s = render.MovingSource(xb, hb, bb, window=(100, 50))
    with pytest.raises(ValueError):
        R.render_host([s], lufs_targets=[-23.0])
    for bad in [(0, 0), (-1, 5), (Nb - 5, 6)]:
        with pytest.raises(ValueError):
            R.render_host([s._replace(window=bad)])
    with pytest.raises(ValueError):
        R.render_host([s], outs=[np.empty((Cb, Nb), np.float32)])
    with pytest.raises(ValueError):
        R.render_host([s._replace(direct_taps=tb)], direct_outs=[np.empty((Cb, Nb), np.float32)])
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ds = render.MovingSource(to(xb), to(hb), to(bb), bb, window=(100, 50))
    with pytest.raises(ValueError):
        R.render_device([ds], [torch.empty((Cb, Nb), device="cuda")])
    with pytest.raises(ValueError):
        R.plan_device([ds], [torch.empty((Cb, 49), device="cuda")])
    R.render_device([ds], [torch.empty((Cb, 50), device="cuda")])
    torch.cuda.synchronize()
