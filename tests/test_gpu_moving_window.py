"""Moving windows (ss_source.win_start_dev; Python: a CUDA int32 tensor as the window's start) through the real kernels.
One plan per case and flag set is run many times with the start tensor rewritten on the stream between runs, without a
host synchronise; every window equals, bit for bit, the slice of the full stem the same plan renders, inside a
NaN-filled output with sentinels on both sides.  Also ss_render_dev with the same items, the graph and its launch
count, sources sharing one start element, a mixed batch whose whole and fixed-window stems keep their bits, clamped
out-of-range starts with bit 2 of ss_device_errors, and the argument checks."""
import ctypes

import numpy as np
import pytest
import torch

from window_cases import CASES, _host_aligned, full_blocks, make_case
from gpu_plumbing import _error_bits, _lib

pytestmark = pytest.mark.gpu

SENT = 1234.5
PAD = 37
# flag set: (SS_RIR_NORMALIZE, SS_DIRECT_TARGET, RIR bank); the banked set uses a bank with normalised taps and a
# direct set, so that the source renders both stems from it
FLAGS = {"plain": (False, False, False), "normalize": (True, False, False), "direct": (False, True, False),
         "bank": (True, True, True)}


class Out:
    """A (C, n) output inside a NaN-filled device buffer with sentinels on both sides."""

    def __init__(self, C, n):
        self.C, self.n = C, n
        self.buf = torch.full((C * n + 2 * PAD,), float("nan"), device="cuda")
        self.buf[:PAD] = SENT
        self.buf[-PAD:] = SENT

    def ptr(self):
        return self.buf.data_ptr() + 4 * PAD

    def reset(self):
        self.buf[PAD:-PAD].fill_(float("nan"))

    @staticmethod
    def stem(snap, C, n, what):
        a = snap.cpu().numpy() if isinstance(snap, torch.Tensor) else snap
        assert np.all(a[:PAD] == SENT) and np.all(a[-PAD:] == SENT), what
        v = a[PAD:-PAD].reshape(C, n)
        assert not np.isnan(v).any(), what
        return v


class Case:
    """The device inputs of one case of window_cases and the ss_source items over them."""

    def __init__(self, name, flagset, host_visible=True):
        L_, R = _lib()
        self.name = name
        self.mode, self.P, self.C, self.Lr, self.N, taps = CASES[name]
        x, h, idx, w, bounds, _ = make_case(name)
        self.bounds = bounds
        normalize, direct, banked = FLAGS[flagset]
        self.direct = direct
        self.taps = taps if direct else 0
        self.raw_norm = normalize and not banked
        self.flags = (L_.SS_RIR_NORMALIZE if self.raw_norm else 0) | (L_.SS_DIRECT_TARGET if direct else 0)
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        self.dx, self.dh = to(x), to(h)
        self.bank = None
        if banked:
            self.bank = ctypes.c_void_p()
            L_.check(R.lib.ss_bank_create_dev(R.ctx, self.dh.data_ptr(), self.P, self.C, self.Lr,
                                              L_.SS_RIR_NORMALIZE | L_.SS_DIRECT_TARGET, taps, None,
                                              ctypes.byref(self.bank)))
        self.db = to(bounds) if self.mode == 1 else None
        self.bh = np.ascontiguousarray(bounds, np.int32) if self.mode == 1 and host_visible else None
        self.di, self.dw = (to(idx), to(w)) if self.mode == 2 else (None, None)
        self.aligned = _host_aligned(self.mode, self.P, self.C, self.Lr, self.N, bounds) if host_visible else \
            int(self.mode == 1 and self.Lr <= 4096 and (self.P - 1) * 4096 <= self.N)

    def item(self, outs, n=0, start_ptr=None, fixed=0):
        L_, _ = _lib()
        it = L_.SsSource(x=self.dx.data_ptr(), N=self.N, P=self.P, C=self.C, L=self.Lr, mode=self.mode,
                         flags=self.flags)
        if self.bank is not None:
            it.rir_bank = self.bank.value
        else:
            it.rir = self.dh.data_ptr()
        it.out = outs[0].ptr()
        if self.direct:
            it.out_direct = outs[1].ptr()
            it.direct_taps = self.taps
        if self.mode == 1:
            it.bounds = self.db.data_ptr()
            if self.bh is not None:
                it.bounds_host = self.bh.ctypes.data
        elif self.mode == 2:
            it.idx, it.w = self.di.data_ptr(), self.dw.data_ptr()
        if n:
            it.win_len, it.win_start = n, fixed
            if start_ptr is not None:
                it.win_start_dev = start_ptr
        return it

    def outs(self, n):
        return [Out(self.C, n) for _ in range(2 if self.direct else 1)]

    def launches(self):
        """Kernel launches per run of a one-chunk plan with a moving window: k_blocks, k_prepare, the render kernel,
        and k_rir_absmax / k_rir_direct for raw RIRs with SS_RIR_NORMALIZE / SS_DIRECT_TARGET."""
        return 3 + int(self.raw_norm) + int(self.direct and self.bank is None)

    def close(self):
        if self.bank is not None:
            _lib()[1].lib.ss_bank_destroy(self.bank)
            self.bank = None


def _starts(case, n, seed):
    """Starts of a window of n samples: 0, N - n, the block and waypoint boundaries +-1 (for the window's first and last
    sample) and random ones, inside [0, N - n]."""
    N = case.N
    blocks = full_blocks(N, case.bounds if case.mode == 1 else None, case.aligned)
    cand = {0, N - n}
    edges = [b[0] for b in blocks] + ([int(v) for v in case.bounds] if case.mode == 1 else [])
    for e in edges:
        cand |= {e - 1, e, e + 1, e - n - 1, e - n, e - n + 1}
    rng = np.random.default_rng(seed)
    cand |= {int(v) for v in rng.integers(0, N - n + 1, 6)}
    return sorted(v for v in cand if 0 <= v <= N - n)


def _lengths(N):
    return [1, min(N, 4096 + 7), N // 3]


def _snap_all(outs):
    return [o.buf.clone() for o in outs]


@pytest.mark.parametrize("flagset", list(FLAGS))
@pytest.mark.parametrize("name", list(CASES))
def test_plan_with_moving_windows(name, flagset):
    L_, R = _lib()
    _error_bits()
    case = Case(name, flagset)
    try:
        lens = _lengths(case.N)
        starts_of = [_starts(case, n, 17 + j) for j, n in enumerate(lens)]
        runs = max(len(s) for s in starts_of)
        table = np.array([[s[k % len(s)] for s in starts_of] for k in range(runs)], np.int32)
        d_table = torch.from_numpy(table).cuda()
        starts = torch.zeros(len(lens), dtype=torch.int32, device="cuda")
        full = case.outs(case.N)
        wouts = [case.outs(n) for n in lens]
        items = [case.item(full)] + [case.item(o, n, starts[j].data_ptr()) for j, (o, n) in enumerate(zip(wouts, lens))]
        arr = (L_.SsSource * len(items))(*items)
        plan = ctypes.c_void_p()
        L_.check(R.lib.ss_plan_create(R.ctx, arr, len(items), ctypes.byref(plan)))
        try:
            snaps = []
            for k in range(runs):                      # no host synchronise inside the loop
                starts.copy_(d_table[k])
                for o in full + sum(wouts, []):
                    o.reset()
                L_.check(R.lib.ss_plan_run(plan, None))
                snaps.append((_snap_all(full), [_snap_all(o) for o in wouts]))
            torch.cuda.synchronize()
            assert R.lib.ss_plan_is_graph(plan) == 1
            ref = [Out.stem(s, case.C, case.N, name) for s in snaps[0][0]]
            for k, (fs, ws) in enumerate(snaps):
                for f, r in zip(fs, ref):
                    assert np.array_equal(Out.stem(f, case.C, case.N, name), r), (name, k)
                for j, n in enumerate(lens):
                    a = int(table[k, j])
                    for stem, r in zip(ws[j], ref):
                        assert np.array_equal(Out.stem(stem, case.C, n, name), r[:, a:a + n]), (name, flagset, n, a)
            # launches of one run, as documented for a chunk that holds a moving window
            R.lib.ss_reset_stats(R.ctx)
            L_.check(R.lib.ss_plan_run(plan, None))
            assert R.lib.ss_launch_count(R.ctx) == case.launches()
            # ss_render_dev with the same items
            for k in (0, runs // 2, runs - 1):
                starts.copy_(d_table[k])
                for o in sum(wouts, []):
                    o.reset()
                L_.check(R.lib.ss_render_dev(R.ctx, arr, len(items), None))
                torch.cuda.synchronize()
                for j, n in enumerate(lens):
                    a = int(table[k, j])
                    for o, r in zip(wouts[j], ref):
                        assert np.array_equal(Out.stem(o.buf, case.C, n, name), r[:, a:a + n]), ("dev", name, n, a)
            assert _error_bits() == 0
        finally:
            R.lib.ss_plan_destroy(plan)
    finally:
        case.close()


@pytest.mark.parametrize("name", ["bounds", "indexed", "static2", "long8"])
def test_out_of_range_starts_are_clamped(name):
    L_, R = _lib()
    _error_bits()
    case = Case(name, "plain")
    n = 5000
    N = case.N
    full, wout = case.outs(N), case.outs(n)
    start = torch.zeros(1, dtype=torch.int32, device="cuda")
    items = (L_.SsSource * 2)(case.item(full), case.item(wout, n, start.data_ptr()))
    plan = ctypes.c_void_p()
    L_.check(R.lib.ss_plan_create(R.ctx, items, 2, ctypes.byref(plan)))
    try:
        L_.check(R.lib.ss_plan_run(plan, None))
        torch.cuda.synchronize()
        ref = Out.stem(full[0].buf, case.C, N, name)
        for v in [-5, N - n + 3, N, 2 ** 31 - 1, -2 ** 31, N - n, 0, 1234]:
            start.fill_(v)
            wout[0].reset()
            L_.check(R.lib.ss_plan_run(plan, None))
            bad = v < 0 or v > N - n
            assert _error_bits() == (4 if bad else 0), v            # reported once ...
            assert _error_bits() == 0, v                            # ... and cleared by the read
            a = min(max(v, 0), N - n)
            assert np.array_equal(Out.stem(wout[0].buf, case.C, n, name), ref[:, a:a + n]), (name, v)
    finally:
        R.lib.ss_plan_destroy(plan)
        case.close()


def test_python_api_shared_starts_and_mixed_batch():
    """A scene's stems share one start element of a (B,) tensor; whole and fixed-window stems in the same plan keep the
    bits of the plan without moving windows; plan_device and render_device agree; check_device_errors reports a
    clamped start."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    _error_bits()
    x, h, idx, w, bounds, taps = make_case("bounds")
    N, C = x.shape[0], h.shape[1]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dx, dh, db = to(x), to(h), to(bounds)
    bank = R.rir_bank(dh)
    n, fixed = 4096 + 11, 1234
    starts = torch.zeros(3, dtype=torch.int32, device="cuda")
    A = render.MovingSource(dx, dh, db, bounds)                          # whole stems
    F = render.StaticSource(dx, dh[0])
    Bk = render.MovingSource(dx, bank, db)                               # banked, trajectory on the device only
    fixed_srcs = [A, A._replace(window=(fixed, n)), F]
    moving = lambda k: [A._replace(window=(starts[k], n)), F._replace(window=(starts[k], n)),
                        Bk._replace(window=(starts[k], n))]
    shape = lambda s: (C, N if s.window is None else s.window[1])
    o_ref = [torch.empty(shape(s), device="cuda") for s in fixed_srcs + [Bk]]
    R.render_device(fixed_srcs + [Bk], o_ref)
    p_fixed = R.plan_device(fixed_srcs, [torch.empty(shape(s), device="cuda") for s in fixed_srcs])
    batch = fixed_srcs[:2] + moving(1) + fixed_srcs[2:] + moving(2)[:1]
    outs = [torch.empty(shape(s), device="cuda") for s in batch]
    plan = R.plan_device(batch, outs)
    hist = []
    for k in range(8):
        starts.copy_(torch.randint(0, N - n + 1, (3,), dtype=torch.int32, device="cuda"))
        plan.run()
        p_fixed.run()
        hist.append((starts.clone(), [o.clone() for o in outs], [o.clone() for o in p_fixed._keep[1]]))
    torch.cuda.synchronize()
    assert plan.is_graph()
    ref_A, ref_Af, ref_F, ref_B = [t.cpu().numpy() for t in o_ref]
    for st, got, fx in hist:
        s1, s2 = int(st[1]), int(st[2])
        got = [t.cpu().numpy() for t in got]
        fx = [t.cpu().numpy() for t in fx]
        want = [ref_A, ref_Af, ref_A[:, s1:s1 + n], ref_F[:, s1:s1 + n], ref_B[:, s1:s1 + n], ref_F,
                ref_A[:, s2:s2 + n]]
        for k, (g, wv) in enumerate(zip(got, want)):
            assert np.array_equal(g, wv), k
        for g, f in zip([got[0], got[1], got[5]], fx):                   # whole and fixed-window stems keep their bits
            assert np.array_equal(g, f)
    assert np.array_equal(ref_Af, ref_A[:, fixed:fixed + n])
    # one chunk holding moving windows: k_blocks, k_prepare, k_render_fast
    c0 = R.launch_count()
    plan.run()
    torch.cuda.synchronize()
    assert R.launch_count() - c0 == 3
    # render_device with the same sources
    starts.copy_(torch.tensor([5, N - n, 77], dtype=torch.int32))
    d_outs = [torch.empty_like(o) for o in outs]
    R.render_device(batch, d_outs)
    plan.run()
    torch.cuda.synchronize()
    for d, o in zip(d_outs, outs):
        assert torch.equal(d, o)
    assert np.array_equal(outs[2].cpu().numpy(), ref_A[:, N - n:])
    R.check_device_errors()
    # a clamped start is reported once
    starts[1] = N
    plan.run()
    with pytest.raises(ValueError):
        R.check_device_errors()
    R.check_device_errors()
    assert np.array_equal(outs[2].cpu().numpy(), ref_A[:, N - n:])
    plan.close()
    p_fixed.close()
    bank.close()


def test_argument_checks():
    from sonicsim_b200 import render
    L_, R = _lib()
    case = Case("bounds", "plain")
    n = 100
    out = case.outs(n)
    start = torch.zeros(4, dtype=torch.int32, device="cuda")
    good = case.item(out, n, start.data_ptr())
    one = lambda it: (L_.SsSource * 1)(it)
    plan = ctypes.c_void_p()
    bad = []
    for field, v in (("win_len", 0), ("win_start", 5), ("win_start_dev", start.data_ptr() + 2)):
        it = case.item(out, n, start.data_ptr())
        setattr(it, field, v)
        bad.append(it)
    for it in bad:
        assert R.lib.ss_render_dev(R.ctx, one(it), 1, None) == L_.SS_ERR_INVALID
        assert R.lib.ss_plan_create(R.ctx, one(it), 1, ctypes.byref(plan)) == L_.SS_ERR_INVALID
    # the host path cannot copy a read set that depends on a start only the device knows
    x = np.ascontiguousarray(make_case("bounds")[0])
    h = np.ascontiguousarray(make_case("bounds")[1])
    host_out = np.full((case.C, n), 7.0, np.float32)
    hb = np.ascontiguousarray(case.bounds, np.int32)
    hit = L_.SsSource(x=x.ctypes.data, rir=h.ctypes.data, out=host_out.ctypes.data, bounds=hb.ctypes.data, N=case.N,
                      P=case.P, C=case.C, L=case.Lr, mode=L_.SS_MOVING_BOUNDS, win_len=n,
                      win_start_dev=start.data_ptr())
    assert R.lib.ss_render_host(R.ctx, one(hit), 1) == L_.SS_ERR_INVALID
    assert np.all(host_out == 7.0)
    L_.check(R.lib.ss_render_dev(R.ctx, one(good), 1, None))
    torch.cuda.synchronize()
    # the Python layer
    src = render.MovingSource(x, h, case.bounds, window=(start[0], n))
    with pytest.raises(ValueError):
        R.render_host([src])
    with pytest.raises(ValueError):
        R.plan_host([src])
    dsrc = render.MovingSource(case.dx, case.dh, case.db, window=(start[0], n))
    o = [torch.empty((case.C, n), device="cuda")]
    for s in (start[:2], start.long()[0], start.cpu()[0], start.float()[0]):
        with pytest.raises(ValueError):
            R.render_device([dsrc._replace(window=(s, n))], o)
        with pytest.raises(ValueError):
            R.plan_device([dsrc._replace(window=(s, n))], o)
    with pytest.raises(ValueError):
        R.plan_device([dsrc], [torch.empty((case.C, n + 1), device="cuda")])
    R.plan_device([dsrc], o).run()
    R.render_device([dsrc._replace(window=(start[1:2], n))], o)
    torch.cuda.synchronize()
    case.close()
