"""RIR spectrum banks through the real kernels.  A source that names a bank renders bit-identically to the same source
given its raw RIRs - through ss_render_host (default context and one with a 1 MB host pipeline budget), ss_render_dev
with and without bounds_host, a device plan run twice with the dry signal changed, and the Python API - for whole stems
and windows, plain / normalised / direct / both.  The banked items carry rir = NULL, the buffer the bank was built from
is NaN once the bank is built, and every output lies between sentinels.  Also: one bank shared by many sources across
chunks, host- and device-built banks, loudness targets, the launches an all-banked batch saves, configs[1] against the
oracle, and every refusal."""
import ctypes

import numpy as np
import pytest
import torch

from chunk_budget import chunk_budget  # noqa: F401  (fixture)
from conftest import TOL
from oracle import sonicsim_oracle as so
from window_cases import CASES, make_case, windows
from gpu_plumbing import _lib, small_host_budget_context

pytestmark = pytest.mark.gpu

SENT = np.float32(1234.5)
PAD = 37
FLAGS = [(False, False), (True, False), (False, True), (True, True)]
FLAG_IDS = ["plain", "normalize", "direct", "normalize+direct"]


def make_bank(ctx, h, normalize, taps, dev=False):
    """An ss_bank of h (P, C, L) built from a copy of h that is NaN-filled right after (host or device creation)."""
    L, R = _lib()
    P, C, Lr = h.shape
    flags = (L.SS_RIR_NORMALIZE if normalize else 0) | (L.SS_DIRECT_TARGET if taps else 0)
    b = ctypes.c_void_p()
    if dev:
        t = torch.from_numpy(np.array(h, np.float32)).cuda()
        L.check(R.lib.ss_bank_create_dev(ctx, t.data_ptr(), P, C, Lr, flags, taps, None, ctypes.byref(b)))
        t.fill_(float("nan"))                   # same (legacy default) stream: after the bank's kernels
        torch.cuda.synchronize()
    else:
        raw = np.array(h, np.float32)
        L.check(R.lib.ss_bank_create_host(ctx, raw.ctypes.data, P, C, Lr, flags, taps, ctypes.byref(b)))
        raw[:] = np.nan
    return b


class Stems:
    """One case rendered as [full source] + [one windowed source per window], raw RIRs or a bank, every output in a
    padded buffer with sentinels."""

    def __init__(self, name, normalize, direct, dev, host_visible, wins, bank=None, x=None):
        L_, _ = _lib()
        mode, P, C, Lr, N, taps = CASES[name]
        x0, h, idx, w, bounds, _ = make_case(name)
        self.C, self.N, self.dev, self.wins = C, N, dev, list(wins)
        flags = (L_.SS_RIR_NORMALIZE if normalize and bank is None else 0) | (L_.SS_DIRECT_TARGET if direct else 0)
        arr = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()) if dev else np.ascontiguousarray
        ptr = (lambda a: a.data_ptr()) if dev else (lambda a: a.ctypes.data)
        self.dx = arr(np.array(x0 if x is None else x, np.float32))
        self.keep = [self.dx]
        dh = arr(h) if bank is None else None
        self.keep.append(dh)
        self.items, self.outs = [], []
        for win in [None] + self.wins:
            n = N if win is None else win[1]
            bufs = []
            for _ in range(2 if direct else 1):
                b = np.full(C * n + 2 * PAD, np.nan, np.float32)
                b[:PAD] = SENT
                b[-PAD:] = SENT
                bufs.append(arr(b))
            it = L_.SsSource(x=ptr(self.dx), rir=ptr(dh) if dh is not None else None, N=N, P=P, C=C, L=Lr, mode=mode,
                             flags=flags)
            if bank is not None:
                it.rir_bank = bank.value
            it.out = ptr(bufs[0]) + 4 * PAD
            if direct:
                it.out_direct = ptr(bufs[1]) + 4 * PAD
                it.direct_taps = taps
            if mode == 1:
                db = arr(bounds)
                it.bounds = ptr(db)
                if host_visible and dev:
                    hb = np.ascontiguousarray(bounds, np.int32)
                    it.bounds_host = hb.ctypes.data
                    self.keep.append(hb)
                self.keep.append(db)
            elif mode == 2:
                di, dw = arr(idx), arr(w)
                it.idx, it.w = ptr(di), ptr(dw)
                self.keep += [di, dw]
            if win is not None:
                it.win_start, it.win_len = win
            self.items.append(it)
            self.outs.append((bufs, n))

    def array(self):
        return (self.items[0].__class__ * len(self.items))(*self.items)

    def set_x(self, x2):
        if self.dev:
            self.dx.copy_(torch.from_numpy(np.ascontiguousarray(x2, np.float32)))
        else:
            self.dx[:] = x2

    def reset(self):
        for bufs, n in self.outs:
            for b in bufs:
                if self.dev:
                    b[PAD:-PAD].fill_(float("nan"))
                else:
                    b[PAD:-PAD] = np.nan

    def stems(self):
        """[[stem (C, n) per output of the item] per item], sentinels checked, every value written."""
        host = (lambda t: t.cpu().numpy()) if self.dev else (lambda t: t)
        res = []
        for bufs, n in self.outs:
            got = []
            for b in bufs:
                a = host(b)
                assert np.all(a[:PAD] == SENT) and np.all(a[-PAD:] == SENT)
                v = a[PAD:-PAD].reshape(self.C, n)
                assert not np.isnan(v).any()
                got.append(v.copy())
            res.append(got)
        return res


def assert_same(a, b, what):
    for k, (sa, sb) in enumerate(zip(a, b)):
        for ga, gb in zip(sa, sb):
            assert np.array_equal(ga, gb), (what, k)


def _wins(name):
    mode, P, C, Lr, N, taps = CASES[name]
    _, _, _, _, bounds, _ = make_case(name)
    return windows(name, N, bounds if mode == 1 else None, 1 if mode == 1 and Lr <= 4096 else 0, seed=5)


def _host(ctx, st):
    L_, R = _lib()
    L_.check(R.lib.ss_render_host(ctx, st.array(), len(st.items)))
    return st.stems()


def _dev(st):
    L_, R = _lib()
    L_.check(R.lib.ss_render_dev(R.ctx, st.array(), len(st.items), None))
    torch.cuda.synchronize()
    return st.stems()


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
@pytest.mark.parametrize("name", list(CASES))
def test_bank_bits_on_every_path(name, flags):
    normalize, direct = flags
    L_, R = _lib()
    mode, P, C, Lr, N, taps = CASES[name]
    h = make_case(name)[1]
    taps = taps if direct else 0
    wins = _wins(name)
    banks = []
    try:
        # host path, default context and 1 MB pipeline chunks (a bank belongs to its context: one per context)
        bank = make_bank(R.ctx, h, normalize, taps)
        banks.append(bank)
        raw = _host(R.ctx, Stems(name, normalize, direct, False, True, wins))
        bst = Stems(name, normalize, direct, False, True, wins, bank)
        assert all(it.rir is None for it in bst.items)
        assert_same(_host(R.ctx, bst), raw, "host")
        with small_host_budget_context() as ctx:
            bank_s = make_bank(ctx, h, normalize, taps)
            try:
                raw = _host(ctx, Stems(name, normalize, direct, False, True, wins))
                assert_same(_host(ctx, Stems(name, normalize, direct, False, True, wins, bank_s)), raw, "host 1 MB")
            finally:
                R.lib.ss_bank_destroy(bank_s)
        # device path with and without bounds_host, a bank built from device memory
        dbank = make_bank(R.ctx, h, normalize, taps, dev=True)
        banks.append(dbank)
        for visible in (True, False):
            raw = _dev(Stems(name, normalize, direct, True, visible, wins))
            assert_same(_dev(Stems(name, normalize, direct, True, visible, wins, dbank)), raw, ("dev", visible))
        bits = ctypes.c_uint32()
        L_.check(R.lib.ss_device_errors(R.ctx, ctypes.byref(bits)))
        assert bits.value == 0
        # a plan, run twice with the dry signal changed in between
        st = Stems(name, normalize, direct, True, True, wins, dbank)
        plan = ctypes.c_void_p()
        L_.check(R.lib.ss_plan_create(R.ctx, st.array(), len(st.items), ctypes.byref(plan)))
        try:
            x2 = so.synth_dry(np.random.default_rng(99), N)
            for k, x in enumerate([None, x2]):
                if k == 1:
                    st.set_x(x2)
                st.reset()
                L_.check(R.lib.ss_plan_run(plan, None))
                torch.cuda.synchronize()
                assert_same(st.stems(), _dev(Stems(name, normalize, direct, True, True, wins, x=x)), ("plan", k))
        finally:
            R.lib.ss_plan_destroy(plan)
    finally:
        for b in banks:
            R.lib.ss_bank_destroy(b)


@pytest.mark.parametrize("name", ["bounds", "static2", "long"])
def test_python_api_banks(name):
    """render_host, plan_host, render_device and plan_device with RirBanks (host- and device-built) against raw RIRs,
    whole stems and windows, with a direct target; a bank with a direct set also serves reverberant-only sources."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    mode, P, C, Lr, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    hb = R.rir_bank(h[0] if mode == 0 else h, direct_taps=taps)
    db = R.rir_bank(to(h[0] if mode == 0 else h), direct_taps=taps)      # used at once: the library orders it
    assert hb.shape == ((C, Lr) if mode == 0 else (P, C, Lr)) and hb.direct_taps == taps and not hb.normalize
    K = (Lr + 4095) // 4096
    assert hb.nbytes == db.nbytes >= 2 * P * C * K * 4096 * 8
    wins = [None] + _wins(name)[1:4]

    def src(r, win, dev=False, taps_=taps):
        t = to if dev else (lambda a: a)
        if mode == 0:
            return render.StaticSource(t(x), r, False, taps_, win)
        return render.MovingSource(t(x), r, t(bounds), bounds if dev else None, False, taps_, win)
    n_of = lambda win: N if win is None else win[1]
    raw_r = [src(h[0] if mode == 0 else h, win) for win in wins]
    rd = [np.empty((C, n_of(win)), np.float32) for win in wins]
    ref = R.render_host(raw_r, direct_outs=rd)
    for bank in (hb, db):
        dd = [np.empty((C, n_of(win)), np.float32) for win in wins]
        outs = R.render_host([src(bank, win) for win in wins], direct_outs=dd)
        hp = R.plan_host([src(bank, win) for win in wins], direct_outs=[np.empty((C, n_of(w_)), np.float32) for w_ in wins])
        pouts = hp.run()
        douts = [torch.empty((C, n_of(win)), device="cuda") for win in wins]
        ddouts = [torch.empty((C, n_of(win)), device="cuda") for win in wins]
        R.render_device([src(bank, win, True) for win in wins], douts, direct_outs=ddouts)
        pl = R.plan_device([src(bank, win, True) for win in wins], [torch.empty((C, n_of(win)), device="cuda") for win in wins],
                           direct_outs=[torch.empty((C, n_of(win)), device="cuda") for win in wins])
        pl.run()
        torch.cuda.synchronize()
        dref = [t.cpu().numpy() for t in douts]
        for k in range(len(wins)):
            assert np.array_equal(outs[k], ref[k]) and np.array_equal(pouts[k], ref[k]), (name, k)
            assert np.array_equal(dd[k], rd[k]), (name, k)
            assert np.array_equal(pl._keep[1][k].cpu().numpy(), dref[k]), (name, k)
            assert np.array_equal(ddouts[k].cpu().numpy(), pl._keep[2][k].cpu().numpy()), (name, k)
        # device path against the device path with raw RIRs
        rdo = [torch.empty((C, n_of(win)), device="cuda") for win in wins]
        R.render_device([src(to(h[0] if mode == 0 else h), win, True) for win in wins], rdo,
                        direct_outs=[torch.empty((C, n_of(win)), device="cuda") for win in wins])
        torch.cuda.synchronize()
        for k in range(len(wins)):
            assert np.array_equal(dref[k], rdo[k].cpu().numpy()), (name, k)
        # a bank with a direct set serves a reverberant-only source
        only = R.render_host([src(bank, None, taps_=0)])[0]
        assert np.array_equal(only, ref[0])
    # host- and device-built banks agree
    assert np.array_equal(R.render_host([src(hb, None)], direct_outs=[np.empty((C, N), np.float32)])[0],
                          R.render_host([src(db, None)], direct_outs=[np.empty((C, N), np.float32)])[0])
    # plans keep their banks alive
    pl = R.plan_host([src(R.rir_bank(h[0] if mode == 0 else h), None, taps_=0)])
    assert np.array_equal(pl.run()[0], R.render_host([src(h[0] if mode == 0 else h, None, taps_=0)])[0])
    hb.close()
    db.close()
    assert hb.closed and db.closed


def test_one_bank_shared_by_many_sources_across_chunks(chunk_budget):  # noqa: F811
    """One bank, 8 sources in one batch, each with its own dry signal and window, cut into several chunks: equal to 8
    separate raw renders."""
    from sonicsim_b200 import render
    R = chunk_budget(1 << 20)
    mode, P, C, Lr, N, taps = CASES["bounds3"]
    _, h, _, _, bounds, _ = make_case("bounds3")
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    bank = R.rir_bank(to(h), direct_taps=taps)
    rng = np.random.default_rng(5)
    xs = [so.synth_dry(rng, N) for _ in range(8)]
    wins = [None, (0, 1), (N - 1, 1), (5000, 4096), (4095, 2), None, (123, 9000), (N // 2, N // 3)]
    n_of = lambda win: N if win is None else win[1]
    srcs = [render.MovingSource(to(x), bank, to(bounds), bounds, False, taps, win) for x, win in zip(xs, wins)]
    outs = [torch.empty((C, n_of(win)), device="cuda") for win in wins]
    douts = [torch.empty((C, n_of(win)), device="cuda") for win in wins]
    n0 = R.launch_count()
    R.render_device(srcs, outs, direct_outs=douts)
    torch.cuda.synchronize()
    assert R.launch_count() - n0 >= 4                  # at least two chunks
    for k, (x, win) in enumerate(zip(xs, wins)):
        o, d = torch.empty((C, n_of(win)), device="cuda"), torch.empty((C, n_of(win)), device="cuda")
        R.render_device([render.MovingSource(to(x), to(h), to(bounds), bounds, False, taps, win)], [o], direct_outs=[d])
        torch.cuda.synchronize()
        assert torch.equal(outs[k], o) and torch.equal(douts[k], d), k


def test_loudness_targets_on_banked_sources():
    from sonicsim_b200 import render
    R = render.default_renderer()
    srcs, banked, shapes = [], [], []
    for name in ("bounds", "static2", "long"):
        mode, P, C, Lr, N, taps = CASES[name]
        x, h, idx, w, bounds, _ = make_case(name)
        r = h[0] if mode == 0 else h
        if mode == 0:
            srcs.append(render.StaticSource(x, r, False, taps))
            banked.append(render.StaticSource(x, R.rir_bank(r, direct_taps=taps), False, taps))
        else:
            srcs.append(render.MovingSource(x, r, bounds, None, False, taps))
            banked.append(render.MovingSource(x, R.rir_bank(r, direct_taps=taps), bounds, None, False, taps))
        shapes.append((C, N))
    targets = [-17.0, -24.0, -29.0]

    def run(ss):
        dd = [np.empty(sh, np.float32) for sh in shapes]
        lo = []
        outs = R.render_host(ss, lufs_targets=targets, loudness_out=lo, direct_outs=dd)
        return outs, dd, lo
    a, ad, al = run(srcs)
    b, bd, bl = run(banked)
    for k in range(3):
        assert np.array_equal(a[k], b[k]) and np.array_equal(ad[k], bd[k]), k
    assert al == bl
    assert all(np.isfinite(v[0]) for v in al)


def test_all_banked_batch_launches_no_rir_kernels():
    """Launch counts: an all-banked batch runs no k_rir_absmax / k_rir_direct (one chunk each here)."""
    L_, R = _lib()
    name = "bounds"
    mode, P, C, Lr, N, taps = CASES[name]
    h = make_case(name)[1]
    for (normalize, direct), saved in zip(FLAGS[1:], (1, 1, 2)):
        bank = make_bank(R.ctx, h, normalize, taps if direct else 0)
        try:
            for dev in (False, True):
                raw = Stems(name, normalize, direct, dev, True, [])
                bst = Stems(name, normalize, direct, dev, True, [], bank)
                render = _dev if dev else (lambda st: _host(R.ctx, st))
                n0 = R.launch_count()
                a = render(raw)
                n1 = R.launch_count()
                b = render(bst)
                n2 = R.launch_count()
                assert (n1 - n0) - (n2 - n1) == saved, (normalize, direct, dev, n1 - n0, n2 - n1)
                assert n2 - n1 == 2
                assert_same(a, b, (normalize, direct, dev))
        finally:
            R.lib.ss_bank_destroy(bank)


def test_cfg2_banked_speakers_against_the_oracle():
    """BASELINE configs[1] speakers (P = 40, C = 6, L = 4096, 30 s at 16 kHz) from a bank, whole and as 4 s crops."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    rng = np.random.default_rng(4243)
    N, C, L, P, sr = 480000, 6, 4096, 40, 16000
    dry, pos, h = so.synth_dry(rng, N), so.synth_path(rng, P), so.synth_rirs(rng, P, C, L)
    np.random.seed(4243)
    bounds = render.trajectory_bounds(pos, N)
    idx = np.repeat(np.arange(P - 1), np.diff(bounds))
    w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(bounds)]).astype(np.float32)
    ref = so.convolve_moving_receiver(dry, h, idx, w)
    bank = R.rir_bank(h)
    assert bank.nbytes >= P * C * 4096 * 8 == 7864320
    wins = [None, (123457, 4 * sr)]
    outs = R.render_host([render.MovingSource(dry, bank, bounds, window=win) for win in wins])
    assert so.rel_rms(outs[0], ref) < TOL
    assert so.rel_rms(outs[1], ref[:, 123457:123457 + 4 * sr]) < TOL


def test_bank_refusals():
    """Every rule of the header, through the C ABI (SS_ERR_INVALID on render_host, render_dev and plan_create) and
    through Python (ValueError before any C call)."""
    from sonicsim_b200 import render
    L_, R = _lib()
    mode, P, C, Lr, N, taps = CASES["bounds"]
    x, h, idx, w, bounds, _ = make_case("bounds")
    bank = make_bank(R.ctx, h, False, 0)
    dbank = make_bank(R.ctx, h, False, taps)
    sbank = make_bank(R.ctx, h[:1], False, 0)
    out = np.zeros((C, N), np.float32)
    outd = np.zeros((C, N), np.float32)
    dx, db, dout, doutd = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (x, bounds, out, outd))
    try:
        def item(dev=False, **kw):
            it = L_.SsSource(x=dx.data_ptr() if dev else x.ctypes.data, out=dout.data_ptr() if dev else out.ctypes.data,
                             bounds=db.data_ptr() if dev else bounds.ctypes.data, N=N, P=P, C=C, L=Lr,
                             mode=L_.SS_MOVING_BOUNDS, rir_bank=bank.value)
            for k, v in kw.items():
                setattr(it, k, v)
            return it
        ok = dict()
        bad = [dict(rir=h.ctypes.data),                                      # rir and rir_bank
               dict(rir_bank=None),                                          # neither
               dict(P=P - 1), dict(C=C + 1), dict(L=Lr + 1),                  # shape
               dict(flags=L_.SS_RIR_NORMALIZE),                              # normalisation belongs to the bank
               dict(flags=L_.SS_DIRECT_TARGET, direct_taps=taps),            # bank without a direct set
               dict(rir_bank=dbank.value, flags=L_.SS_DIRECT_TARGET, direct_taps=taps + 1),
               dict(rir_bank=sbank.value, mode=L_.SS_MOVING_BOUNDS),         # moving source, P = 1 bank
               dict(rir_bank=sbank.value, mode=L_.SS_STATIC, P=1, bounds=None)]   # static source, P = 1 bank: valid
        with small_host_budget_context() as ctx:                              # another context's bank
            other = make_bank(ctx, h, False, 0)
            try:
                for kw, want in [(ok, L_.SS_OK), (dict(rir_bank=other.value), L_.SS_ERR_INVALID)] + \
                        [(k, L_.SS_ERR_INVALID) for k in bad[:-1]] + [(bad[-1], L_.SS_OK)]:
                    hkw, dkw = dict(kw), dict(kw)
                    if kw.get("flags", 0) & L_.SS_DIRECT_TARGET:             # with its output: only the bank rule fails
                        hkw["out_direct"], dkw["out_direct"] = outd.ctypes.data, doutd.data_ptr()
                    got = R.lib.ss_render_host(R.ctx, (L_.SsSource * 1)(item(**hkw)), 1)
                    assert got == want, ("host", kw)
                    ditems = (L_.SsSource * 1)(item(True, **dkw))
                    assert R.lib.ss_render_dev(R.ctx, ditems, 1, None) == want, ("dev", kw)
                    plan = ctypes.c_void_p()
                    assert R.lib.ss_plan_create(R.ctx, ditems, 1, ctypes.byref(plan)) == want, ("plan", kw)
                    R.lib.ss_plan_destroy(plan)
                torch.cuda.synchronize()
            finally:
                R.lib.ss_bank_destroy(other)
        # creation arguments
        b = ctypes.c_void_p()
        for args in [(None, P, C, Lr, 0, 0), (h.ctypes.data, 0, C, Lr, 0, 0), (h.ctypes.data, P, 0, Lr, 0, 0),
                     (h.ctypes.data, P, C, 0, 0, 0), (h.ctypes.data, P, C, Lr, 4, 0),
                     (h.ctypes.data, P, C, Lr, L_.SS_DIRECT_TARGET, 0)]:
            assert R.lib.ss_bank_create_host(R.ctx, *args, ctypes.byref(b)) == L_.SS_ERR_INVALID, args
        assert R.lib.ss_bank_create_host(R.ctx, h.ctypes.data, P, C, Lr, 0, 0, None) == L_.SS_ERR_INVALID
        assert R.lib.ss_bank_create_host(None, h.ctypes.data, P, C, Lr, 0, 0, ctypes.byref(b)) == L_.SS_ERR_INVALID
    finally:
        for bk in (bank, dbank, sbank):
            R.lib.ss_bank_destroy(bk)
    # Python: ValueError before any C call
    rb = R.rir_bank(h, direct_taps=taps)
    s = render.MovingSource(x, rb, bounds)
    R.render_host([s])
    for bad_src in [s._replace(normalize_rirs=True), s._replace(direct_taps=taps + 1),
                    render.MovingSource(x, R.rir_bank(h[:P - 1]), bounds),        # P - 1 positions, P bounds
                    render.StaticSource(x, rb)]:                                   # a static source needs P == 1
        with pytest.raises(ValueError):
            R.render_host([bad_src], direct_outs=[np.empty((C, N), np.float32)] if bad_src.direct_taps else None)
    with pytest.raises(ValueError):                                                # outputs of another C
        R.render_host([s], outs=[np.empty((C + 1, N), np.float32)])
    with small_host_budget_context() as ctx:
        R2 = render.Renderer.__new__(render.Renderer)
        R2.lib, R2.device, R2.ctx = R.lib, R.device, ctx
        foreign = R2.rir_bank(h)
        for call in (lambda: R.render_host([render.MovingSource(x, foreign, bounds)]),
                     lambda: R.plan_device([render.MovingSource(dx, foreign, db, bounds)], [dout])):
            with pytest.raises(ValueError):
                call()
        foreign.close()
    rb.close()
    for call in (lambda: R.render_host([s]), lambda: R.render_device([render.MovingSource(dx, rb, db)], [dout])):
        with pytest.raises(ValueError):
            call()
    with pytest.raises(ValueError):
        R.rir_bank(np.zeros(5, np.float32))
    with pytest.raises(ValueError):
        R.rir_bank(h, direct_taps=-1)


def test_device_built_bank_is_ordered_before_every_use():
    """A bank built from a tensor on a side stream that still has ~0.2 s of queued work is used at once, with no
    synchronisation, by render_host / plan_host (the library's own streams), render_device and a device plan (torch's
    default stream): every stem equals the render from the raw RIRs.  Every bank stays alive to the end, so no bank can
    inherit a finished one's memory."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    mode, P, C, Lr, N, taps = CASES["bounds"]
    x, _, _, _, bounds, _ = make_case("bounds")
    h = so.synth_rirs(np.random.default_rng(2024), P, C, Lr)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ref_d = np.empty((C, N), np.float32)
    ref = R.render_host([render.MovingSource(x, h, bounds, None, True, taps)], direct_outs=[ref_d])[0]
    side = torch.cuda.Stream()
    th = to(h)
    torch.cuda.synchronize()
    banks = []

    def busy_bank():
        with torch.cuda.stream(side):
            torch.cuda._sleep(int(4e8))
            bank = R.rir_bank(th, normalize=True, direct_taps=taps)
        banks.append(bank)
        return bank

    def check(out, out_d, what):
        assert np.array_equal(out, ref) and np.array_equal(out_d, ref_d), what
    b = busy_bank()
    assert not side.query()                           # the bank is still being built when the render starts
    d = np.empty((C, N), np.float32)
    check(R.render_host([render.MovingSource(x, b, bounds, None, False, taps)], direct_outs=[d])[0], d, "render_host")
    b = busy_bank()
    d = np.empty((C, N), np.float32)
    hp = R.plan_host([render.MovingSource(x, b, bounds, None, False, taps)], direct_outs=[d])
    assert not side.query()
    check(hp.run()[0], d, "plan_host")
    b = busy_bank()
    assert not side.query()
    o, od = torch.empty((C, N), device="cuda"), torch.empty((C, N), device="cuda")
    R.render_device([render.MovingSource(to(x), b, to(bounds), bounds, False, taps)], [o], direct_outs=[od])
    torch.cuda.synchronize()
    check(o.cpu().numpy(), od.cpu().numpy(), "render_device")
    b = busy_bank()
    o, od = torch.empty((C, N), device="cuda"), torch.empty((C, N), device="cuda")
    pl = R.plan_device([render.MovingSource(to(x), b, to(bounds), bounds, False, taps)], [o], direct_outs=[od])
    pl.run()
    torch.cuda.synchronize()
    check(o.cpu().numpy(), od.cpu().numpy(), "plan_device")
    pl.close()
    for b in banks:
        b.close()


def test_closing_a_bank_keeps_its_plans_running():
    """close() refuses the bank to new sources at once; plans made before keep rendering from it, and its memory is
    freed when the last of them goes."""
    import gc
    from sonicsim_b200 import render
    R = render.default_renderer()
    mode, P, C, Lr, N, taps = CASES["bounds"]
    x, h, _, _, bounds, _ = make_case("bounds")
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    ref = R.render_host([render.MovingSource(x, h, bounds)])[0]
    bank = R.rir_bank(h)
    o = torch.empty((C, N), device="cuda")
    pl = R.plan_device([render.MovingSource(to(x), bank, to(bounds), bounds)], [o])
    hp = R.plan_host([render.MovingSource(x, bank, bounds)])
    bank.close()
    assert bank.closed and bank._h
    with pytest.raises(ValueError):
        R.render_host([render.MovingSource(x, bank, bounds)])
    o.fill_(float("nan"))
    pl.run()
    torch.cuda.synchronize()
    assert np.array_equal(o.cpu().numpy(), ref)
    assert np.array_equal(hp.run()[0], ref)
    pl.close()
    assert bank._h                                    # the host plan still holds it
    del hp
    gc.collect()
    assert not bank._h
