"""Loudness slots of device plans (render.StemLoudness; ss_stream_lufs) in the kernels' per-thread code, on the CPU:
the gate of k_loud_gate<true>, which reads its target from memory at every run, and k_loud_crop, which cuts a slot's
crop out of its measured whole stem.  Checked against a float64 reference, the host-target gate and oracle lufs_norm:
the gain and its float32 rounding, a silent stem (-inf LUFS gained as -40), NaN and +-inf targets (bit 6, gain 1, result
gain NaN) and the start clamp at both edges (bit 2)."""
import ctypes
import math
import os
import sys

import numpy as np
import pytest

from oracle import sonicsim_oracle as so
from loudness_cases import EXACT_DB, assert_clear_of_gates, block_size_of, stems

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "emu"))
import build_emu  # noqa: E402

RATE = 16000


@pytest.fixture(scope="module")
def lib():
    """tests/emu/ss_emu_stream_loud.cu built by build_emu, with the argtypes of its two entry points."""
    h = ctypes.CDLL(build_emu.build("ss_emu_stream_loud"))
    vp, i32, f64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double
    h.emu_lufs_dev.argtypes = [vp, i32, i32, f64, f64, vp, vp, i32, vp, vp, i32, vp]
    h.emu_loud_crop.argtypes = [vp] * 5 + [i32] * 4 + [vp, vp, ctypes.POINTER(ctypes.c_int32)]
    return h


def ptr(a):
    return a.ctypes.data if a is not None else None


def measure_dev(lib, x, sr, target):
    """(LUFS, gain) of the (N, C) stem x with the target read from memory (k_loud_gate<true>)."""
    from sonicsim_b200.SonicSim_audio import gating_plan
    N, C = x.shape
    cn = np.ascontiguousarray(x.T)
    block = block_size_of(N, sr)
    brk, lo, hi = gating_plan(N, float(sr), float(block))
    t = np.array([target], np.float64)
    res = np.full(2, -7.0)
    lib.emu_lufs_dev(ptr(cn), N, C, float(sr), float(block), ptr(t), ptr(brk), len(brk) - 1, ptr(lo), ptr(hi), len(lo),
                     ptr(res))
    return float(res[0]), float(res[1])


@pytest.mark.parametrize("N,C,sr", [(60000, 2, 16000), (48000, 1, 16000), (100001, 3, 16000), (96000, 5, 48000)])
def test_device_target_gate_matches_the_host_target_gate_and_the_oracle(lib, emu, N, C, sr):
    x = stems(N * 3 + C, N, C, sr)
    block = block_size_of(N, sr)
    assert_clear_of_gates(x, sr, block)
    ref = so.bs1770_integrated_loudness(x, sr, block, up_to_8_channels=True)
    for t in (-17.0, -24.25, -29.0, -19.0 + 1e-9):
        lufs, gain = measure_dev(lib, x, sr, t)
        assert (lufs, gain) == emu.lufs(x, sr, block, target=t)           # the same bits as a target on the host
        assert abs(lufs - ref) <= EXACT_DB, (lufs, ref)
        assert abs(gain / 10 ** ((t - lufs) / 20) - 1) < 1e-12
        y, _ = so.lufs_norm(x, sr, t, up_to_8_channels=True)              # the oracle's float32 stem
        assert np.max(np.abs(x * np.float32(gain) - y)) <= 2e-6 * np.max(np.abs(y))


def test_silent_stem_is_gained_as_minus_40(lib):
    x = np.zeros((32000, 2), np.float32)
    lufs, gain = measure_dev(lib, x, RATE, -24.0)
    assert math.isinf(lufs) and lufs < 0
    assert gain == 10.0 ** ((-24.0 + 40.0) / 20.0)


@pytest.mark.parametrize("target", [math.nan, math.inf, -math.inf])
def test_non_finite_target_leaves_the_gain_nan(lib, target):
    x = stems(5, 32000, 2)
    lufs, gain = measure_dev(lib, x, RATE, target)
    assert lufs == measure_dev(lib, x, RATE, -20.0)[0] and math.isnan(gain)


def crop(lib, whole, whole_dir, start, length, target, result, host_start=0):
    C, N = whole.shape
    out = np.full((C, length), np.nan, np.float32)
    out_d = np.full((C, length), np.nan, np.float32) if whole_dir is not None else None
    ws = np.array([start], np.int32) if start is not None else None
    t = np.array([target], np.float64)
    r = np.asarray(result, np.float64)
    s = ctypes.c_int32(-1)
    err = lib.emu_loud_crop(ptr(whole), ptr(whole_dir), ptr(out), ptr(out_d), ptr(ws), host_start, length, N, C, ptr(t),
                            ptr(r), ctypes.byref(s))
    return out, out_d, err, s.value


@pytest.mark.parametrize("length", [16000, 16001, 4003])
def test_crop_is_the_slice_times_the_float32_gain(lib, length):
    rng = np.random.default_rng(length)
    C, N = 2, 48000
    whole = rng.standard_normal((C, N)).astype(np.float32)
    whole_d = rng.standard_normal((C, N)).astype(np.float32)
    gain = 10 ** ((-17.0 - -31.7) / 20) * (1 + 1e-9)               # not a float32: the crop rounds it once
    g = np.float32(gain)
    assert float(g) != gain
    hi = N - length
    cases = [(0, 0, 0), (hi, hi, 0), (1234, 1234, 0), (-5, 0, 4), (hi + 3, hi, 4), (2 ** 31 - 1, hi, 4),
             (-2 ** 31, 0, 4)]
    for v, s0, bits in cases:
        out, out_d, err, s = crop(lib, whole, whole_d, v, length, -17.0, [-31.7, gain])
        assert (s, err) == (s0, bits)
        assert np.array_equal(out, whole[:, s0:s0 + length] * g)
        assert np.array_equal(out_d, whole_d[:, s0:s0 + length] * g)
        ref = whole[:, s0:s0 + length].astype(np.float64) * gain       # float64 reference: one float32 rounding
        assert np.max(np.abs(out - ref) / np.maximum(np.abs(ref), 1e-30)) <= 2 ** -24 * (1 + 1e-6) + abs(float(g) - gain) / gain
    out, out_d, err, s = crop(lib, whole, None, None, length, -17.0, [-31.7, gain], host_start=77)
    assert (s, err, out_d) == (77, 0, None) and np.array_equal(out, whole[:, 77:77 + length] * g)


@pytest.mark.parametrize("target", [math.nan, math.inf, -math.inf])
def test_crop_with_a_non_finite_target_is_unscaled_with_bit_6(lib, target):
    whole = np.random.default_rng(3).standard_normal((3, 20000)).astype(np.float32)
    out, _, err, s = crop(lib, whole, None, 500, 8000, target, [-20.0, math.nan])
    assert (s, err) == (500, 64) and np.array_equal(out, whole[:, 500:8500])
    out, _, err, s = crop(lib, whole, None, 20000, 8000, target, [-20.0, math.nan])
    assert (s, err) == (12000, 64 | 4) and np.array_equal(out, whole[:, 12000:])
