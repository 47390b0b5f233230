"""Drop-in for the hot-path functions of the reference module SonicSim-SonicSet/SonicSim_audio.py:
`fft_conv` (:17-47), `lufs_norm` (:68-81), `get_lufs_norm_audio` (:83-86).  Same names, argument
meaning, return types and exception types; the arithmetic runs in the CUDA library (C ABI in
include/sonicsim_b200.h).  No CPU fallback.

Dry-stream assembly (:152-340) is re-exported from sonicsim_b200.dry (host logic, same `random` stream as the
reference).  Out of scope (SURVEY section 2): generate_rir_combination (:342-400), which wraps Habitat.

Loudness follows pyloudnorm 0.1.1 (the reference's pin, ss-2.0.yaml:201), restated from its
published algorithm because the package is not vendored in the reference: "parity unpinned".
"""
import ctypes
import functools
import os
import math

import numpy as np

from . import _lib
from .dry import (create_background_audio, create_long_audio, get_random_wav_path,      # noqa: F401  (:152-340, host logic)
                  get_random_wav_path_from_json)


# ------------------------------------------------------------------------------------ loudness
REFINE = int(os.environ.get("SS_LOUD_REFINE", "1"))     # elementary intervals per gating hop: more, shorter recurrences per
                                                         # channel for the K-weighting kernels (experiment knob; measured: no gain,
                                                         # the passes are bound by float64 throughput, not by thread count)


@functools.lru_cache(maxsize=64)
def gating_plan(num_samples: int, rate: float, block_size: float, refine: int = REFINE):
    """Gating-block sample bounds exactly as pyloudnorm 0.1.1 computes them (meter.py: float
    expressions truncated with int(), 75 % overlap), in the compact form the C ABI takes:
    (brk int32[n_e + 1], blk_lo int32[nb], blk_hi int32[nb]).  `brk` holds every distinct block bound plus
    `refine - 1` evenly spaced cut points inside each interval between them: the kernels run one thread per
    (channel, interval) and carry the exact filter state across intervals, so any partition gives the same result -
    a finer one just means more, shorter threads."""
    T_g = block_size
    step = 1.0 - 0.75
    T = num_samples / rate
    num_blocks = int(np.round(((T - T_g) / (T_g * step))) + 1)
    lo = [min(int(T_g * (j * step) * rate), num_samples) for j in range(num_blocks)]
    hi = [min(int(T_g * (j * step + 1) * rate), num_samples) for j in range(num_blocks)]      # x[l:u] clips at N
    brk = np.unique(np.array(lo + hi, dtype=np.int64))
    if refine > 1 and len(brk) > 1:
        a, b = brk[:-1], brk[1:]
        cuts = [a + (b - a) * k // refine for k in range(1, refine)]
        brk = np.unique(np.concatenate([brk] + cuts))
    blk_lo = np.searchsorted(brk, lo).astype(np.int32)
    blk_hi = np.searchsorted(brk, hi).astype(np.int32)
    return brk.astype(np.int32), blk_lo, blk_hi


def gating_block_size(num_samples, rate):
    """SonicSim_audio.py:69: lufs_norm's gating block in seconds, 0.4 or the whole stem when that is shorter."""
    return 0.4 if num_samples / rate >= 0.4 else num_samples / rate


def _valid_audio(data, rate, block_size):
    """pyloudnorm.util.valid_audio."""
    if not isinstance(data, np.ndarray):
        raise ValueError("Data must be of type numpy.ndarray.")
    if not np.issubdtype(data.dtype, np.floating):
        raise ValueError("Data must be floating point.")
    if data.ndim == 2 and data.shape[1] > 5:
        raise ValueError("Audio must have five channels or less.")
    if data.shape[0] < block_size * rate:
        raise ValueError("Audio must have length greater than the block size.")
    return True


def integrated_loudness_and_norm(data: np.ndarray, sr, block_size, target, want_output=True):
    """Measure (and normalise) one stem (N, C) or (N,) on the GPU.  Returns (lufs, gain, out|None)."""
    _valid_audio(data, sr, block_size)
    x = np.ascontiguousarray(data, dtype=np.float32)
    N = x.shape[0]
    C = 1 if x.ndim == 1 else x.shape[1]
    brk, blk_lo, blk_hi = gating_plan(N, float(sr), float(block_size))
    out = np.empty_like(x) if want_output else None
    lufs, gain = ctypes.c_double(), ctypes.c_double()
    st = _lib.load().ss_lufs_norm_host(
        _lib.context(), x.ctypes.data, out.ctypes.data if out is not None else None, N, C,
        C, 1, float(sr), float(block_size), float(target), brk.ctypes.data, len(brk) - 1,
        blk_lo.ctypes.data, blk_hi.ctypes.data, len(blk_lo), ctypes.byref(lufs), ctypes.byref(gain))
    _lib.check(st)
    return lufs.value, gain.value, out


def lufs_norm(data, sr, norm=-6):
    """SonicSim_audio.py:68-81 -> (norm_data, gain)."""
    loudness, _, out = integrated_loudness_and_norm(np.asarray(data), sr, gating_block_size(len(data), sr), norm)
    if math.isinf(loudness):                                                        # :73-75 (applied on the device too)
        print("loudness is inf")
    norm_data = out if np.asarray(data).dtype == np.float32 else out.astype(np.asarray(data).dtype)
    n, d = np.sum(np.array(norm_data)), np.sum(np.array(data))                      # :78
    gain = n / d if d else 0.0                                                      # :79
    return norm_data, gain


def get_lufs_norm_audio(audio, sr=16000, lufs=-6):
    """SonicSim_audio.py:83-86: target ~ U(lufs - 2, lufs + 2) drawn from the global NumPy RNG."""
    class_lufs = np.random.uniform(lufs - 2, lufs + 2)                              # :84
    data_norm, gain = lufs_norm(data=audio, sr=sr, norm=class_lufs)
    return data_norm, gain


# ------------------------------------------------------------------------------------ fft_conv
def fft_conv(signal, kernel, is_cpu: bool = False):
    """SonicSim_audio.py:17-47: zero-pad both to M = N + L - 1, rfftn * rfftn -> irfftn.

    M even: the result is the full linear convolution (length M); it runs on the CUDA renderer as a
    static overlap-save render of the zero-extended signal.
    M odd: the reference calls `irfftn` without a length, which returns M - 1 samples of the
    band-limited interpolant of the convolution resampled at stride M / (M - 1) - not a convolution
    (rel. error 0.7-0.9 against one).  `fft_conv` is dead code on the SonicSet path (SURVEY 8a a6); for
    fidelity this quirk is reproduced with the same torch.fft calls on the CUDA device rather than
    with a kernel of our own."""
    import torch
    from .SonicSim_moving import convolve_fixed_receiver
    dev = signal.device
    n_sig, n_ker = signal.numel(), kernel.numel()
    if (n_sig + n_ker - 1) % 2 == 1:
        import torch.nn.functional as F
        if not torch.cuda.is_available():
            raise RuntimeError("sonicsim_b200.fft_conv needs a CUDA device (no CPU fallback)")
        s = F.pad(signal.detach().reshape(-1).to("cuda", torch.float32), (0, n_ker - 1))
        k = F.pad(kernel.detach().reshape(-1).to("cuda", torch.float32), (0, n_sig - 1))
        out = torch.fft.irfftn(torch.fft.rfftn(s, dim=-1) * torch.fft.rfftn(k, dim=-1), dim=-1)
        return out.cpu() if is_cpu else out.to(dev)
    x = signal.detach().reshape(-1).to("cpu", torch.float32).numpy()
    h = kernel.detach().reshape(-1).to("cpu", torch.float32).numpy()
    xp = np.concatenate([x, np.zeros(h.shape[0] - 1, np.float32)])
    y = convolve_fixed_receiver(xp[None, :], h[None, :])[0]
    out = torch.from_numpy(y)
    return out if is_cpu else out.to(dev)


# ------------------------------------------------------------------------------------ small helpers
def normalize(audio, norm="peak"):
    """SonicSim_audio.py:49-66."""
    if norm == "peak":
        peak = abs(audio).max()
        return audio / peak if peak != 0 else audio
    if norm == "rms":
        if hasattr(audio, "numpy"):
            audio = audio.numpy()
        rms = np.sqrt(np.mean(np.square(np.trim_zeros(audio, trim="b")))) * 100
        return audio / rms if rms != 0 else audio
    raise NotImplementedError
