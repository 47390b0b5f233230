"""RIR spectrum banks on the CPU: the emulation (tests/emu/ss_emu_bank.cu) builds a bank with the kernels' own
k_rir_absmax / k_rir_direct / k_prepare phases over a source without blocks, and renders banked sources through the
kernels' own fill_items and render CTAs.  Every banked render equals, bit for bit, the emulated render of the same source
given its raw RIRs - whole stems against the full and dual emulations, windows against emu_render_window - for plain,
normalised, direct and normalised + direct banks, with the raw RIR buffer NaN-filled once the bank is built.  Also the
Python layer's refusals that need no device."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from window_cases import CASES, KSPEC, _p, make_case, windows


@pytest.fixture(scope="module")
def bank_emu():
    return build_emu.load("ss_emu_bank")


def create(lib, h, normalize, taps):
    """(spec (sets, P*C*K, 4096) complex64, cut (P*C,) or None) of the RIR set h (P, C, L)."""
    P, C, L = h.shape
    K = (L + 4095) // 4096
    sets = 2 if taps else 1
    spec = np.full((sets, P * C * K, KSPEC), np.nan, np.complex64)
    cut = np.full(P * C, -1, np.int32) if taps else None
    n = lib.emu_bank_create(_p(h), P, C, L, int(normalize), int(taps), _p(spec), _p(cut))
    assert n == sets * ((P * C * K + 1) // 2)
    assert not np.isnan(spec.view(np.float32)).any()
    return spec, cut


def banked(lib, x, spec, cut, mode, P, C, L, aligned, win=(0, 0), idx=None, w=None, bounds=None, taps=0):
    N = x.shape[0]
    n = win[1] or N
    out = np.full((C, n), np.nan, np.float32)
    out_d = np.full((C, n), np.nan, np.float32) if taps else None
    stats = np.zeros(3, np.int32)
    lib.emu_render_banked(_p(x), _p(spec), _p(cut), _p(out), _p(bounds), _p(idx), _p(w), N, P, C, L, mode,
                          int(aligned), win[0], win[1], _p(out_d), int(taps), _p(stats))
    assert stats[0] == 0                       # a banked source transforms no RIR row
    return out, out_d


def raw_whole(lib, x, h, mode, idx, w, bounds, taps, normalize):
    """The emulated render of the source given its raw RIRs: emu_render, or emu_render_dual with a direct target or
    normalisation (its `out` is the reverberant stem with the same bits)."""
    P, C, L = h.shape
    N = x.shape[0]
    out, out_d = np.zeros((C, N), np.float32), np.zeros((C, N), np.float32)
    if not taps and not normalize:
        lib.emu_render(_p(x), _p(h), _p(out), _p(bounds), _p(idx), _p(w), N, P, C, L, mode)
        return out, None
    lib.emu_render_dual(_p(x), _p(h), _p(out), _p(bounds), _p(idx), _p(w), N, P, C, L, mode, _p(out_d),
                        int(taps or 1), int(normalize))
    return out, (out_d if taps else None)


def raw_window(lib, x, h, win, mode, aligned, idx, w, bounds, taps, normalize):
    P, C, L = h.shape
    N = x.shape[0]
    out, out_d = np.full((C, win[1]), np.nan, np.float32), np.full((C, win[1]), np.nan, np.float32)
    lib.emu_render_window(_p(x), _p(h), _p(out), _p(bounds), _p(idx), _p(w), N, P, C, L, mode, int(aligned),
                          win[0], win[1], _p(out_d), int(taps), int(normalize), 1, None)
    return out, (out_d if taps else None)


def _kw(mode, idx, w, bounds):
    return dict(idx=idx if mode == 2 else None, w=w if mode == 2 else None, bounds=bounds if mode == 1 else None)


FLAGS = [(False, False), (True, False), (False, True), (True, True)]
FLAG_IDS = ["plain", "normalize", "direct", "normalize+direct"]


@pytest.mark.parametrize("flags", FLAGS, ids=FLAG_IDS)
@pytest.mark.parametrize("name", list(CASES))
def test_emu_banked_render_equals_raw_render(bank_emu, name, flags):
    normalize, direct = flags
    mode, P, C, L, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    taps = taps if direct else 0
    aligned = 1 if mode == 1 and L <= 4096 else 0
    kw = _kw(mode, idx, w, bounds)
    raw = np.array(h, np.float32, copy=True)
    spec, cut = create(bank_emu, raw, normalize, taps)
    raw[:] = np.nan                             # the bank keeps nothing of the buffer it was built from
    # whole stem against the full / dual emulation of the raw source
    ref, ref_d = raw_whole(bank_emu, x, h, mode, kw["idx"], kw["w"], kw["bounds"], taps, normalize)
    out, out_d = banked(bank_emu, x, spec, cut, mode, P, C, L, aligned, taps=taps, **kw)
    assert np.array_equal(out, ref), name
    if direct:
        assert np.array_equal(out_d, ref_d), name
    # windows against the emulated windowed render of the raw source
    for win in windows(name, N, bounds if mode == 1 else None, aligned):
        ref, ref_d = raw_window(bank_emu, x, h, win, mode, aligned, kw["idx"], kw["w"], kw["bounds"], taps, normalize)
        out, out_d = banked(bank_emu, x, spec, cut, mode, P, C, L, aligned, win, taps=taps, **kw)
        assert np.array_equal(out, ref), (name, win)
        if direct:
            assert np.array_equal(out_d, ref_d), (name, win)


@pytest.mark.parametrize("name", ["bounds3", "static3", "long1"])
def test_emu_bank_direct_set_follows_the_reverberant_set(bank_emu, name):
    """A bank with a direct set holds the plain bank's spectra first (one set stride = P*C*K rows), so it also serves
    sources that render only the reverberant stem."""
    mode, P, C, L, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    plain, _ = create(bank_emu, h, False, 0)
    dual, cut = create(bank_emu, h, False, taps)
    assert np.array_equal(dual[0].view(np.float32), plain[0].view(np.float32))
    from direct_path import direct_path_rirs
    cut_ref = np.minimum(L, np.abs(h).argmax(axis=-1) + taps).reshape(-1)
    assert np.array_equal(cut, cut_ref)
    assert np.array_equal(direct_path_rirs(h, taps)[0, 0, :cut[0]], h[0, 0, :cut[0]])
    aligned = 1 if mode == 1 and L <= 4096 else 0
    kw = _kw(mode, idx, w, bounds)
    a, _ = banked(bank_emu, x, plain, None, mode, P, C, L, aligned, **kw)
    b, _ = banked(bank_emu, x, dual, cut, mode, P, C, L, aligned, **kw)
    assert np.array_equal(a, b)


def test_python_refuses_bad_bank_use_before_any_c_call():
    """The checks of render._bank_of that need no device: closed bank, other context, shape, normalize_rirs and
    direct_taps.  (A stand-in renderer / bank: nothing here reaches the library.)"""
    from sonicsim_b200 import render

    class FakeRenderer:
        def __init__(self, ctx):
            self.ctx = ctypes.c_void_p(ctx)

    class FakeBank(render.RirBank):
        def __init__(self, renderer, shape, normalize=False, direct_taps=0, handle=1):
            self.renderer, self._h = renderer, ctypes.c_void_p(handle)
            self.shape, self.normalize, self.direct_taps, self.nbytes = shape, normalize, direct_taps, 0
            self._closing, self._plans = False, 0

        def _free(self):
            self._h = ctypes.c_void_p()
    R, other = FakeRenderer(1000), FakeRenderer(2000)
    x = np.zeros(100, np.float32)
    b = np.array([0, 50, 100], np.int32)
    ok = FakeBank(R, (3, 2, 300), direct_taps=40)
    assert render._bank_of(R, render.MovingSource(x, ok, b), 0, 3, 2, 300) == 1
    assert render._bank_of(R, render.MovingSource(x, ok, b, direct_taps=40), 0, 3, 2, 300) == 1
    assert render._bank_of(R, render.StaticSource(x, FakeBank(R, (2, 300))), 0, 1, 2, 300) == 1
    bad = [
        (render.MovingSource(x, FakeBank(other, (3, 2, 300)), b), (3, 2, 300)),          # another context
        (render.MovingSource(x, ok, b), (3, 2, 301)),                                     # shape
        (render.StaticSource(x, FakeBank(R, (2, 2, 300))), (1, 2, 300)),                  # static needs P == 1
        (render.MovingSource(x, ok, b, normalize_rirs=True), (3, 2, 300)),
        (render.MovingSource(x, ok, b, direct_taps=41), (3, 2, 300)),
        (render.MovingSource(x, FakeBank(R, (3, 2, 300)), b, direct_taps=40), (3, 2, 300)),   # no direct set
    ]
    closed = FakeBank(R, (3, 2, 300))
    closed.close()
    bad.append((render.MovingSource(x, closed, b), (3, 2, 300)))
    for s, pcl in bad:
        with pytest.raises(ValueError):
            render._bank_of(R, s, 0, *pcl)


def test_closing_a_bank_waits_for_the_plans_that_use_it():
    """RirBank.close() refuses the bank to new sources at once, but frees it only when the last plan holding it is
    closed or collected.  (Stand-in bank and plans: the bookkeeping is pure Python.)"""
    import gc
    from sonicsim_b200 import render
    freed = []

    class Bank(render.RirBank):
        def __init__(self):
            self._h, self._closing, self._plans, self.shape = ctypes.c_void_p(1), False, 0, (3, 2, 300)

        def _free(self):
            if self._h:
                freed.append(self)
                self._h = ctypes.c_void_p()

    class Plan:
        pass
    x, b = np.zeros(100, np.float32), np.array([0, 50, 100], np.int32)
    bank, other = Bank(), Bank()
    srcs = [render.MovingSource(x, bank, b), render.MovingSource(x, bank, b), render.StaticSource(x, other)]
    p1, p2 = Plan(), Plan()
    fin1, p2._fin = render._hold_banks(p1, srcs), render._hold_banks(p2, srcs[:1])
    assert bank._plans == 2 and other._plans == 1
    bank.close()
    assert bank.closed and bank._h and not freed            # refused to new sources, still held by two plans
    fin1()                                                   # p1 closed: the plan releases its banks once
    fin1()
    assert bank._plans == 1 and not freed and other._plans == 0 and not other.closed
    del p2
    gc.collect()                                             # p2 collected: the last holder is gone
    assert freed == [bank] and bank.closed
    other.close()
    assert freed == [bank, other]
