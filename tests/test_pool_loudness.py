"""Loudness gains of source pools (ss_pool_loudness) on the CPU: the emulated kernels (tests/emu/ss_emu_gain.cu, the same
phases with the gain handed to fill_items as k_prepare hands it stem_gain) store exactly the ungained output times the
float32 gain, rounded once, in every epilogue branch - static pairs with and without a partner channel, single-segment
blocks under aligned and grid blocking, blocks that straddle waypoints (the red_add branch), indexed trajectories, long
RIRs, windows and direct stems; with gain 1 every output keeps its bits; the head of k_blocks carries the picked
candidate's gain into the slot; the export and version; and the refusals Python makes before any C call."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from sonicsim_b200 import _lib

B = 4096


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_gain")


@pytest.fixture(scope="module")
def emu_plain():
    return build_emu.load("ss_emu_window")


def _addr(a):
    return a.ctypes.data if a is not None else None


def _case(name):
    """(x, rir, bounds, idx, w, N, P, C, L, mode, aligned, window, taps) of one emulated source."""
    rng = np.random.default_rng(108 + CASES.index(name))
    x = rng.standard_normal(3 * B + 1234).astype(np.float32)
    N = len(x)
    bounds = idx = w = None
    if name in ("static3", "static2"):
        C, L, P, mode, aligned = (3 if name == "static3" else 2), 700, 1, 0, 0
        rir = rng.standard_normal((C, L)).astype(np.float32) * 0.1
    else:
        C, L = 2, (5000 if name == "long" else 900)
        if name in ("aligned", "long", "window"):
            P = 4
            bounds = np.round(np.linspace(0, N, P)).astype(np.int32)
        else:                                            # grid: many segments shorter than a block
            P = 9
            bounds = np.concatenate([[0], np.sort(rng.integers(1, N, P - 2)), [N]]).astype(np.int32)
        mode = 1
        aligned = int(name in ("aligned", "window"))
        if name == "indexed":
            mode = 2
            counts = np.diff(bounds)
            idx = np.repeat(np.arange(P - 1), counts).astype(np.int32)
            w = np.concatenate([np.arange(c) / c for c in counts]).astype(np.float32)
        rir = rng.standard_normal((P, C, L)).astype(np.float32) * 0.1
    window = (1500, 2 * B + 77) if name == "window" else (0, 0)
    taps = 40 if name in ("window", "grid") else 0
    return x, rir, bounds, idx, w, N, P, C, L, mode, aligned, window, taps


CASES = ["static3", "static2", "aligned", "grid", "indexed", "long", "window"]


def _render(lib, case):
    x, rir, bounds, idx, w, N, P, C, L, mode, aligned, (ws, wl), taps = case
    T = wl if wl else N
    out = np.full((C, T), np.nan, np.float32)
    dout = np.full((C, T), np.nan, np.float32) if taps else None
    lib.emu_render_window(_addr(x), _addr(rir), _addr(out), _addr(bounds), _addr(idx), _addr(w), N, P, C, L, mode,
                          aligned, ws, wl, _addr(dout), taps, 0, 1, None)
    return out, dout


def _straddles(case):
    """Grid blocks that meet more than one trajectory segment: their samples take the red_add branch."""
    _, _, bounds, _, _, N, P, _, _, mode, aligned, _, _ = case
    if mode == 0 or aligned:
        return 0
    return sum(len(set(np.searchsorted(bounds, [s, min(s + B, N) - 1], side="right"))) > 1 for s in range(0, N, B))


@pytest.mark.parametrize("name", CASES)
def test_gain_scales_every_store_once(emu, emu_plain, name):
    case = _case(name)
    emu.emu_set_gain(1.0)
    base, dbase = _render(emu, case)
    plain, dplain = _render(emu_plain, case)
    assert not np.isnan(base).any()
    assert np.array_equal(base.view(np.uint32), plain.view(np.uint32)), name          # gain 1: the same bits
    if dbase is not None:
        assert np.array_equal(dbase.view(np.uint32), dplain.view(np.uint32)), name
    if name in ("grid", "indexed"):
        assert _straddles(case) > 0, name
    for g in (np.float32(0.3712), np.float32(7.25), np.float32(1e-3), np.nextafter(np.float32(1), np.float32(2))):
        emu.emu_set_gain(float(g))
        out, dout = _render(emu, case)
        want = (base * g).astype(np.float32)                                            # one float32 multiply
        assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), (name, g)
        if dbase is not None:                                                           # the direct stem: same gain
            assert np.array_equal(dout.view(np.uint32), (dbase * g).astype(np.float32).view(np.uint32)), (name, g)
    emu.emu_set_gain(1.0)


def test_pick_slot_carries_the_gain(emu):
    gains = np.array([0.5, 2.0, np.float32(1.0000001), 3.25], np.float32)
    out = np.zeros(2, np.int32)
    g = ctypes.c_float()
    for v, want, bad in [(0, 0, 0), (2, 2, 0), (3, 3, 0), (4, 3, 1), (-5, 0, 1)]:
        emu.emu_pick_slot(v, 4, gains.ctypes.data, out.ctypes.data, ctypes.byref(g))
        assert out.tolist() == [want, bad], v
        assert np.float32(g.value) == gains[want], v
        emu.emu_pick_slot(v, 4, None, out.ctypes.data, ctypes.byref(g))
        assert out.tolist() == [want, bad] and g.value == 1.0, v


def test_pool_loudness_is_exported():
    lib = ctypes.CDLL(_lib.build())
    assert hasattr(lib, "ss_pool_loudness") and "ss_pool_loudness" in _lib.EXPORTS
    assert lib.ss_version() == 108
    loaded = _lib.load()
    assert loaded.ss_pool_loudness(None, None) == _lib.SS_ERR_INVALID


@pytest.mark.parametrize("targets, sr, match", [
    ([-17.0], 16000, "entries in lufs_targets"),
    ([-17.0, None, -20.0, -1.0], 16000, "entries in lufs_targets"),
    ([-17.0, float("nan"), None], 16000, "not finite"),
    ([float("inf"), -17.0, None], 16000, "not finite"),
    ([-17.0, None, -20.0], 0, "sr must be > 0"),
    ([-17.0, None, -20.0], -16000, "sr must be > 0"),
])
def test_source_pool_refuses_bad_targets_before_any_call(targets, sr, match):
    """Checked before the candidates are even looked at (and so before any C call)."""
    from sonicsim_b200 import render
    fake = object.__new__(render.Renderer)               # no context: a C call would fail differently
    with pytest.raises(ValueError, match=match):
        render.Renderer.source_pool(fake, [object(), object(), object()], lufs_targets=targets, sr=sr)
