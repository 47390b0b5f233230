"""Time windows on the CPU: the emulated kernels (tests/emu/ss_emu_window.cu: the same blocking, pairing, item-filling
and epilogue code as the CUDA kernels) render a window equal, bit for bit, to the same samples of the emulated full
render; the window reads nothing outside its documented read set; ss_debug_plan's windowed table is the stated subset of
the full plan; and the argument checks of the pure-host hooks and of the Python layer."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from window_cases import CASES, _bad_bounds, full_blocks, make_case, poison, read_set, windows
from sonicsim_b200 import _lib


@pytest.fixture(scope="module")
def render_window():
    """emu_render_window of tests/emu/ss_emu_window.cu, built with g++ like the other emulation libraries."""
    lib = build_emu.load("ss_emu_window")
    fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int32)

    def ptr(a, t=fp):
        return a.ctypes.data_as(t) if a is not None else None

    def render(x, h, win, mode, aligned, idx=None, w=None, bounds=None, taps=0, normalize=False, restrict=True,
               dual_fn=None):
        x, h = np.ascontiguousarray(x, np.float32), np.ascontiguousarray(h, np.float32)
        P, C, L = h.shape
        N = x.shape[0]
        a, n = win
        out, out_d = np.full((C, n), np.nan, np.float32), np.full((C, n), np.nan, np.float32)
        idx = None if idx is None else np.ascontiguousarray(idx, np.int32)
        w = None if w is None else np.ascontiguousarray(w, np.float32)
        bounds = None if bounds is None else np.ascontiguousarray(bounds, np.int32)
        stats = np.zeros(4, np.int32)
        lib.emu_render_window(ptr(x), ptr(h), ptr(out), ptr(bounds, ip), ptr(idx, ip), ptr(w), N, P, C, L, mode,
                              int(aligned), a, n, ptr(out_d), int(taps), int(normalize), int(restrict),
                              ptr(stats, ip))
        return out, (out_d if taps else None), stats

    def dual(x, h, mode, idx=None, w=None, bounds=None, taps=0, normalize=False):
        x, h = np.ascontiguousarray(x, np.float32), np.ascontiguousarray(h, np.float32)
        P, C, L = h.shape
        N = x.shape[0]
        out, out_d = np.zeros((C, N), np.float32), np.zeros((C, N), np.float32)
        lib.emu_render_dual(ptr(x), ptr(h), ptr(out), ptr(bounds, ip), ptr(idx, ip), ptr(w), N, P, C, L, mode,
                            ptr(out_d), int(taps), int(normalize))
        return out, out_d
    render.dual = dual
    return render


def _kw(mode, idx, w, bounds):
    return dict(idx=idx, w=w) if mode == 2 else dict(bounds=bounds if mode == 1 else None)


def _plans(name):
    """(mode, blocking plans to emulate): bounds sources with one RIR partition both ways."""
    mode, P, C, L, N, taps = CASES[name]
    return mode, ([1, 0] if mode == 1 and L <= 4096 else [0])


@pytest.mark.parametrize("flags", [(False, False), (True, True)], ids=["plain", "normalize+direct"])
@pytest.mark.parametrize("name", list(CASES))
def test_emu_window_equals_full_render_slice(emu, render_window, name, flags):
    normalize, direct = flags
    mode, P, C, L, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    taps = taps if direct else 0
    kw = _kw(mode, idx, w, bounds)
    aligned_default = 1 if mode == 1 and L <= 4096 else 0
    for aligned in _plans(name)[1]:
        full, full_d, st = render_window(x, h, (0, N), mode, aligned, taps=taps, normalize=normalize, **kw)
        if aligned == aligned_default:               # the whole window is the existing emulated render
            if direct or normalize:
                ref, ref_d = render_window.dual(x, h, mode, taps=taps if direct else 1, normalize=normalize, **kw)
                assert np.array_equal(full, ref)
                if direct:
                    assert np.array_equal(full_d, ref_d)
            else:
                assert np.array_equal(full, emu.render(x, h, mode=mode, **kw))
        for win in windows(name, N, bounds if mode == 1 else None, aligned):
            a, n = win
            out, out_d, st = render_window(x, h, win, mode, aligned, taps=taps, normalize=normalize, **kw)
            assert np.array_equal(out, full[:, a:a + n]), (name, aligned, win)
            if direct:
                assert np.array_equal(out_d, full_d[:, a:a + n]), (name, aligned, win)
            # the emulated table and RIR rows are the documented read set's
            K = (L + 4095) // 4096
            rs = read_set(mode, P, C, L, N, bounds, aligned, win)
            kept = [b for b in full_blocks(N, bounds if mode == 1 else None, aligned) if b[0] < a + n and b[0] + b[1] > a]
            assert st[1] == len(kept)
            assert st[2] % 2 == 0
            assert st[2] // (C * K) == rs[2][0] and (st[2] + st[3] - 1) // (C * K) == rs[2][1]


@pytest.mark.parametrize("name", ["bounds", "bounds3", "indexed", "static3", "long1", "zeroseg"])
def test_emu_window_reads_only_its_read_set(render_window, name):
    mode, P, C, L, N, taps = CASES[name]
    x, h, idx, w, bounds, _ = make_case(name)
    aligned = 1 if mode == 1 and L <= 4096 else 0
    kw = _kw(mode, idx, w, bounds)
    for win in windows(name, N, bounds if mode == 1 else None, aligned, seed=1)[1:]:
        ref, ref_d, _ = render_window(x, h, win, mode, aligned, taps=taps, **kw)
        rs = read_set(mode, P, C, L, N, bounds, aligned, win)
        x2, h2, idx2, w2 = poison(x, h, idx if mode == 2 else None, w if mode == 2 else None, rs)
        kw2 = _kw(mode, idx2, w2, bounds)
        out, out_d, _ = render_window(x2, h2, win, mode, aligned, taps=taps, **kw2)
        assert np.array_equal(out, ref), (name, win, rs)
        assert np.array_equal(out_d, ref_d), (name, win, rs)


def test_emu_window_without_host_trajectory_transforms_every_row(render_window):
    """A device-side trajectory (no bounds_host): every RIR row is transformed, the bits stay those of the full render."""
    x, h, idx, w, bounds, taps = make_case("bounds3")
    N = x.shape[0]
    full, full_d, _ = render_window(x, h, (0, N), 1, 1, bounds=bounds, taps=taps)
    for win in windows("bounds3", N, bounds, 1):
        out, out_d, st = render_window(x, h, win, 1, 1, bounds=bounds, taps=taps, restrict=False)
        assert st[2] == 0 and st[3] == h.shape[0] * h.shape[1]
        assert np.array_equal(out, full[:, win[0]:win[0] + win[1]])
        assert np.array_equal(out_d, full_d[:, win[0]:win[0] + win[1]])


def _debug_plan(N, P, L, bounds, win=(0, 0), mode=_lib.SS_MOVING_BOUNDS):
    lib = _lib.load()
    b = np.ascontiguousarray(bounds, dtype=np.int32) if bounds is not None else None
    item = _lib.SsSource(x=1, rir=1, out=1, bounds=b.ctypes.data if b is not None else None, N=N, P=P, C=2, L=L,
                         mode=mode, bounds_host=b.ctypes.data if b is not None else None,
                         win_start=win[0], win_len=win[1])
    cap = (N + 4095) // 4096 + P
    out = np.zeros((cap, 4), dtype=np.int32)
    aligned = ctypes.c_int32(-1)
    n = lib.ss_debug_plan(ctypes.byref(item), out.ctypes.data, cap, ctypes.byref(aligned))
    return (out[:n] if n >= 0 else n), aligned.value


def test_debug_plan_window_is_the_subset_of_the_full_plan():
    rng = np.random.default_rng(11)
    saw = set()
    for case in range(150):
        P = int(rng.integers(2, 60))
        N = int(rng.integers(P, 150000))
        if case % 3 == 0:                          # many short segments: the cost rule picks the grid
            cuts = np.sort(rng.integers(0, min(N, 3000) + 1, P - 2))
        else:
            cuts = np.sort(rng.integers(0, N + 1, P - 2))
        bounds = np.concatenate([[0], cuts, [N]]).astype(np.int32)
        L = int(rng.choice([300, 4096, 4097]))
        full, aligned = _debug_plan(N, P, L, bounds)
        saw.add(aligned)
        for _ in range(4):
            a = int(rng.integers(0, N))
            n = int(rng.integers(1, N - a + 1))
            got, al = _debug_plan(N, P, L, bounds, (a, n))
            assert al == aligned
            want = full[(full[:, 0] < a + n) & (full[:, 0] + full[:, 1] > a)]
            assert np.array_equal(got, want), (case, a, n)
    assert saw == {0, 1}
    # static and indexed sources: the grid
    full, _ = _debug_plan(20000, 1, 300, None, mode=_lib.SS_STATIC)
    got, _ = _debug_plan(20000, 1, 300, None, (4095, 2), mode=_lib.SS_STATIC)
    assert np.array_equal(got, full[:2])


def test_window_argument_checks():
    bounds = np.array([0, 5000, 10000], np.int32)
    ok, _ = _debug_plan(10000, 3, 300, bounds, (9999, 1))
    assert len(ok) == 1
    for win in [(0, -1), (-1, 5), (3, 0), (9000, 1001), (1, 10000), (0x7fffffff, 0x7fffffff)]:
        got, _ = _debug_plan(10000, 3, 300, bounds, win)
        assert got == _lib.SS_ERR_INVALID, win
    # the Python layer refuses before any C call
    from sonicsim_b200 import render
    src = render.MovingSource(np.zeros(100, np.float32), np.zeros((3, 1, 4), np.float32), bounds)
    for win in [(0, 0), (-1, 5), (50, 51), (100, 1)]:
        with pytest.raises(ValueError):
            render._window(src._replace(window=win), 0, 100)
    assert render._window(src._replace(window=(99, 1)), 0, 100) == (99, 1, 1)
    assert render._window(src, 0, 100) == (0, 0, 100)


def test_debug_plan_refuses_bounds_outside_the_contract():
    """The block planner runs only on a validated bounds table: every invalid one is SS_ERR_INVALID, windowed or not."""
    N = 40960
    good, bad = _bad_bounds(N)
    P = len(good)
    for win in [(0, 0), (5000, 64000 // 16), (0, N)]:
        got, _ = _debug_plan(N, P, 300, good.astype(np.int32), win)
        assert not isinstance(got, int) and len(got) > 0
        for b in bad:
            got, _ = _debug_plan(N, P, 300, b.astype(np.int32), win)
            assert got == _lib.SS_ERR_INVALID, (b, win)
