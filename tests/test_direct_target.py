"""Direct-path target (SS_DIRECT_TARGET) on the CPU: the NumPy definition against the per-row recipe, and the emulated
kernels (tests/emu, the same per-thread code as the CUDA kernels) rendering both stems of a source in one pass against
rendering each RIR set as a source of its own, bit for bit."""
import ctypes

import numpy as np
import pytest

from conftest import TOL
from direct_path import CASES, direct_path_rirs, make_case, normalized, oracle_render
from emu import build_emu
from oracle import sonicsim_oracle as so


@pytest.fixture(scope="module")
def render_dual():
    """emu_render_dual of tests/emu/ss_emu_dual.cu, built with g++ like the other emulation library."""
    lib = build_emu.load("ss_emu_dual")
    fp, ip = ctypes.POINTER(ctypes.c_float), ctypes.POINTER(ctypes.c_int32)

    def ptr(a, t=fp):
        return a.ctypes.data_as(t) if a is not None else None

    def render(x, h, taps, idx=None, w=None, bounds=None, mode=2, normalize=False):
        x, h = np.ascontiguousarray(x, np.float32), np.ascontiguousarray(h, np.float32)
        P, C, L = h.shape
        N = x.shape[0]
        out, out_d = np.zeros((C, N), np.float32), np.zeros((C, N), np.float32)
        idx = None if idx is None else np.ascontiguousarray(idx, np.int32)
        w = None if w is None else np.ascontiguousarray(w, np.float32)
        bounds = None if bounds is None else np.ascontiguousarray(bounds, np.int32)
        lib.emu_render_dual(ptr(x), ptr(h), ptr(out), ptr(bounds, ip), ptr(idx, ip), ptr(w), N, P, C, L, mode,
                            ptr(out_d), int(taps), int(normalize))
        return out, out_d
    return render


def _loop_recipe(h, taps):
    """test_cfg5_binaural_dual_render's construction of the direct RIR set."""
    peak = np.abs(h).argmax(axis=-1)
    hd = h.copy()
    for p in range(h.shape[0]):
        for c in range(h.shape[1]):
            hd[p, c, peak[p, c] + taps:] = 0
    return hd


def test_direct_path_rirs_equals_loop_recipe():
    rng = np.random.default_rng(5000)
    h = so.synth_rirs(rng, 40, 2, 4096)
    assert np.array_equal(direct_path_rirs(h, int(0.0025 * 16000)), _loop_recipe(h, 40))
    for name in CASES:
        _, h, _, _, _, taps = make_case(name)
        assert np.array_equal(direct_path_rirs(h, taps), _loop_recipe(h, taps)), name
        for t in (1, 7, h.shape[-1] + 5):
            assert np.array_equal(direct_path_rirs(h, t), _loop_recipe(h, t)), (name, t)


def test_special_rows_cut_where_the_definition_says():
    _, h, _, _, _, taps = make_case("static3")
    L = h.shape[-1]
    hd = direct_path_rirs(h, taps)
    assert hd[0, 0, L // 3] != 0 and not hd[0, 0, L // 3 + taps:].any()             # tie: the first maximum wins
    assert np.array_equal(hd[0, 1], h[0, 1])                                       # peak near the end: cut = L
    assert not hd[0, 2].any()                                                      # all-zero row


def _ref_stems(emu, x, h, idx, w, bounds, mode, taps, normalize):
    hr = normalized(h) if normalize else h
    kw = dict(idx=idx, w=w, mode=mode) if mode == 2 else dict(bounds=bounds, mode=mode)
    hr2 = hr[0] if mode == 0 else hr
    hd = direct_path_rirs(hr, taps)
    return emu.render(x, hr2, **kw), emu.render(x, hd[0] if mode == 0 else hd, **kw), hr, hd


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("name", list(CASES))
def test_emu_dual_equals_two_separate_sources(emu, render_dual, name, normalize):
    x, h, idx, w, bounds, taps = make_case(name)
    mode = CASES[name][0]
    kw = dict(idx=idx, w=w, mode=mode) if mode == 2 else dict(bounds=bounds, mode=mode)
    out, out_d = render_dual(x, h, taps, normalize=normalize, **kw)
    ref, ref_d, hr, hd = _ref_stems(emu, x, h, idx, w, bounds, mode, taps, normalize)
    assert np.array_equal(out, ref)
    assert np.array_equal(out_d, ref_d)
    assert not np.array_equal(out, out_d)
    assert so.rel_rms(out_d, oracle_render(x, hd, idx, w)) < TOL
    assert so.rel_rms(out, oracle_render(x, hr, idx, w)) < TOL


def normalisation_tie_rirs(taps):
    """Static (C = 2, L = 1000) RIRs whose row 1 holds two taps a < b that divide by the global abs-max (3, in row 0)
    to the same float32: on raw taps b is the peak, on normalised taps the earlier a."""
    m = np.float32(3.0)
    a = np.float32(1.5)
    while a / m != np.nextafter(a, np.float32(2)) / m:                       # search the first colliding neighbours
        a = np.nextafter(a, np.float32(2))
    b = np.nextafter(a, np.float32(2))
    rng = np.random.default_rng(77)
    h = (rng.standard_normal((1, 2, 1000)) * 0.1).astype(np.float32)
    h[0, 0, 5] = m
    h[0, 1, 10], h[0, 1, 200] = a, b
    assert a < b and a / m == b / m
    assert np.abs(h[0, 1]).argmax() == 200 and np.abs(normalized(h)[0, 1]).argmax() == 10
    assert not np.array_equal(direct_path_rirs(normalized(h), taps), normalized(direct_path_rirs(h, taps)))
    return h


def test_emu_normalisation_tie_takes_the_first_normalised_peak(emu, render_dual):
    taps = 40
    h = normalisation_tie_rirs(taps)
    x = so.synth_dry(np.random.default_rng(78), 9000)
    out, out_d = render_dual(x, h, taps, mode=0, normalize=True)
    ref, ref_d, _, hd = _ref_stems(emu, x, h, None, None, None, 0, taps, True)
    assert not hd[0, 1, 50:].any() and hd[0, 1, 10] != 0
    assert np.array_equal(out, ref)
    assert np.array_equal(out_d, ref_d)
