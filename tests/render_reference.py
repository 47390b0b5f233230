"""Float64 restatement of the render (k_prepare + k_render / k_render_fast), the local float32 rounding scale of an
overlap-save output sample, a sample-by-sample check of a rendered stem against both, and structured inputs that turn
a local fault (a wrong sample position, hat weight, block end, dry window, partition offset or history) into a large
local error.  Import-only.

A global relative RMS over a whole stem cannot see a fault confined to a few samples per block: one wrong hat weight
at every block end moves the RMS of a 30 s stem by about 2e-6.  check_render therefore bounds every sample's error by
the rounding scale of the transforms that produce it (error_scale), and the global RMS only as a second check."""
import math

import numpy as np
from scipy import ndimage, signal

from oracle import sonicsim_oracle as so

B = 4096            # overlap-save block = RIR partition length (csrc/ss_core.cuh kB)
F = 8192            # FFT length (kF)

# Bounds of check_render, calibrated on the CPU emulation of the kernels (tests/test_emu_parity.py: about 8x the worst
# ratios the emulated kernels reach over its structured inputs and shape edges, 3.0e-6 and 5.2e-7).
TAU_LOCAL = 2.5e-5   # max |y - y64| / scale of any sample
TAU_GLOBAL = 3e-6   # relative RMS of a stem against float64


def trajectory(bounds):
    """(idx, w) of a compact trajectory: what setup_dynamic_interp gives for these segment bounds (np.repeat of the
    segment counts, np.linspace(0, 1, n_s, endpoint=False) per segment as float32).  Empty segments get no samples."""
    n = np.diff(np.asarray(bounds, np.int64))
    idx = np.repeat(np.arange(n.size), n)
    w = np.concatenate([np.zeros(0)] + [np.linspace(0, 1, k, endpoint=False) for k in n]).astype(np.float32)
    return idx, w


def bounds_from_lengths(lengths):
    """int32 cumulative segment bounds (P,) of segments of the given lengths (0: an empty segment)."""
    return np.concatenate([[0], np.cumsum(np.asarray(lengths, np.int64))]).astype(np.int32)


def _pcl(h):
    h = np.asarray(h)
    return h[None] if h.ndim == 2 else h


def render_f64(x, h, mode, bounds=None, idx=None, w=None, window=None):
    return _render_f64(x, h, mode, bounds, idx, w, window)[0]


def _render_f64(x, h, mode, bounds=None, idx=None, w=None, window=None):
    """The stem of one source in float64, (C, N) - or (C, n) for window = (a, n): output samples [a, a + n).
    mode 0: static, h (C, L) or (1, C, L); mode 1: compact trajectory `bounds` (P,); mode 2: per-sample (idx, w).
    Segment-local form (so.convolve_moving_exact_f64): y[c, n] = (1 - w[n]) (x * h[idx[n], c])[n] + w[n]
    (x * h[idx[n] + 1, c])[n], each position's convolution by fftconvolve in float64, with the hat weights the reference
    and the kernels use: w[n] and 1 - w[n] rounded to float32 (SonicSim_moving.py:94 on a float32 w).  A window convolves
    only x[a - L + 1 : a + n], which is all those samples depend on, so a window of a full-size stem costs only the
    window.

    _render_f64 also returns the envelope |conv_idx[n]| + |conv_idx[n]+1| (static: |conv| of the channel and of its
    transform partner), the magnitudes an inverse transform that makes sample n holds."""
    x = np.asarray(x, np.float64).reshape(-1)
    h = _pcl(np.asarray(h, np.float64))
    N, L = x.size, h.shape[-1]
    a, n = (0, N) if window is None else (int(window[0]), int(window[1]))
    a0 = max(0, a - L + 1)
    xs = x[a0:a + n]
    if mode == 0:
        y = signal.fftconvolve(xs[None], h[0], mode="full")[:, a - a0:xs.size]
        env = np.abs(y)
        return y, np.maximum(env, env[np.minimum(np.arange(env.shape[0]) ^ 1, env.shape[0] - 1)])
    if mode == 1:
        idx, w = trajectory(bounds)
    idx = np.asarray(idx, np.int64)[a0:a + n]
    w1 = np.asarray(w, np.float32)[a0:a + n]
    w0 = (np.float32(1) - w1).astype(np.float64)
    w1 = w1.astype(np.float64)
    y = np.zeros((h.shape[1], xs.size))
    env = np.zeros_like(y)
    for p in np.unique(np.concatenate([idx, idx + 1])):
        s0, s1 = idx == p, idx + 1 == p
        conv = signal.fftconvolve(xs[None], h[p], mode="full")[:, :xs.size]
        y[:, s0] += w0[s0] * conv[:, s0]
        y[:, s1] += w1[s1] * conv[:, s1]
        s = s0 | s1
        env[:, s] += np.abs(conv[:, s])
    return y[:, a - a0:], env[:, a - a0:]


def positions_of(mode, bounds=None, idx=None):
    """Per-sample first position idx[n] of the lerp (None for a static source), the `positions` of error_scale."""
    if mode == 0:
        return None
    return trajectory(bounds)[0] if mode == 1 else np.asarray(idx, np.int64)


def error_scale(x, h, positions=None, window=None):
    """Local float32 rounding scale of every output sample, (C, N) (or (C, n) for window = (a, n)):

        scale(c, n) = sum_j ||x[n - 4096 (j + 3), n - 4096 j + 8192)||_2 * max_{p, c'} ||h[p, c', j-th partition]||_2 / sqrt(8192)

    x clipped to [0, N).  A sample of block start s is made by inverse transforms of the dry windows
    x[s - 4096 (j + 1), s - 4096 j + 4096), s in (n - 4096, n]; each dry window shares its forward transform with a
    neighbouring block's window and carries that partner's rounding error, hence one more block on either side.
    (p, c') runs over the RIR rows whose error reaches sample n of channel c: the positions idx[n] - 1 .. idx[n] + 2
    (two per inverse transform, a grid block pairs them from its first position on; {0} for a static source), channel c
    and its transform partner (static: channels 2k, 2k + 1), and every RIR row's forward-transform partner (rows
    2r, 2r + 1 of the (P, C, K) list).  So silence, sparse RIRs and quiet stretches cannot raise false alarms, and a
    local fault cannot hide behind the stem's RMS.  `positions`: positions_of(...)."""
    x = np.asarray(x, np.float64).reshape(-1)
    h = _pcl(np.asarray(h, np.float64))
    P, C, L = h.shape
    N, K = x.size, -(-L // B)
    a, n = (0, N) if window is None else (int(window[0]), int(window[1]))
    hp = np.zeros((P, C, K))
    for j in range(K):
        hp[:, :, j] = np.sqrt(np.sum(h[:, :, j * B:(j + 1) * B] ** 2, axis=-1))
    rows = hp.reshape(-1)
    partner = np.minimum(np.arange(rows.size) ^ 1, rows.size - 1)
    hp = np.maximum(rows, rows[partner]).reshape(P, C, K)
    if positions is None:                                        # static: channels 2k, 2k + 1 share a transform
        pair = np.minimum(np.arange(C) ^ 1, C - 1)
        hp = np.maximum(hp, hp[:, pair])
    cs = np.concatenate([[0.0], np.cumsum(x * x)])
    nn = np.arange(a, a + n)
    scale = np.zeros((C, n))
    for j in range(K):
        lo, hi = np.clip(nn - B * (j + 3), 0, N), np.clip(nn - B * j + 2 * B, 0, N)
        xn = np.sqrt(np.maximum(cs[hi] - cs[lo], 0.0))
        if positions is None:
            hm = np.repeat(hp[0, :, j][:, None], n, axis=1)
        else:
            p = np.asarray(positions, np.int64)[a:a + n]
            hm = np.zeros((C, n))
            for d in (-1, 0, 1, 2):
                q = np.clip(p + d, 0, P - 1)
                hm = np.maximum(hm, hp[q, :, j].T)
        scale += xn[None] * hm
    return scale / math.sqrt(F)


def render_check_inputs(x, h, mode, bounds=None, idx=None, w=None, window=None):
    """(y64, scale) of one source: render_f64 and the scale check_render divides by,

        error_scale + env[c, n] + max_{|m - n| < 8192} env[c, m] / 8 + 2^-30 max |y64|,

    env the envelope of _render_f64 (both convolutions the lerp of sample n reads, both channels of a static pair).
    The second and third terms matter where the output is sparse (an impulse train through pure-delay RIRs), where a
    norm over 20480 samples spreads a few large samples thin: the lerp and the store round in proportion to the
    convolutions they combine, and the late passes of the inverse transform in proportion to the largest outputs of the
    transform (real and imaginary part).  The last one is the float64 reference's own rounding, which is all there is
    where the exact output is 0."""
    y64, env = _render_f64(x, h, mode, bounds, idx, w, window)
    if not y64.size:
        return y64, env
    peak = ndimage.maximum_filter1d(env, size=2 * F - 1, axis=1, mode="constant")
    scale = error_scale(x, h, positions_of(mode, bounds, idx), window) + env + peak / 8
    return y64, scale + np.abs(y64).max() * 2.0 ** -30


def local_ratio(y, y64, scale):
    """|y - y64| / scale per sample; where the scale is 0 (no signal reaches the sample) the error must be exactly 0."""
    err = np.abs(np.asarray(y, np.float64) - np.asarray(y64, np.float64))
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(scale > 0, err / np.where(scale > 0, scale, 1.0), np.where(err > 0, np.inf, 0.0))


def check_render(y, y64, scale, tau_local, tau_global, n0=0, label=""):
    """Assert that a rendered stem y (C, n) holding output samples [n0, n0 + n) meets its float64 reference y64 sample by
    sample - max |y - y64| / scale <= tau_local over every 4096-sample tile of the output grid - and as a whole - global
    relative RMS <= tau_global.  Returns (worst local ratio, global relative RMS) for the caller to report.  A stem whose
    float64 reference is silent to float64 rounding (RMS under 2^-20 of the scale's, e.g. N shorter than the RIRs' onset)
    has no meaningful relative RMS; its global error is taken relative to the RMS of the scale instead."""
    y = np.asarray(y, np.float64)
    y64 = np.asarray(y64, np.float64)
    assert y.shape == y64.shape == scale.shape, (label, y.shape, y64.shape, scale.shape)
    assert np.all(np.isfinite(y)), "%s: non-finite output samples at %s" % (label, np.argwhere(~np.isfinite(y))[:4].tolist())
    if y.size == 0:
        return 0.0, 0.0
    def rms(v):
        return math.sqrt(float(np.mean(v * v)))
    den = rms(y64)
    if den < rms(scale) * 2.0 ** -20:
        den = rms(scale)
    g = rms(y - y64) / den if den > 0 else rms(y - y64)
    r = local_ratio(y, y64, scale)
    c, i = np.unravel_index(int(np.argmax(r)), r.shape)
    worst = float(r[c, i])
    if worst > tau_local:
        tiles = (n0 + np.arange(y.shape[1])) // B
        bad = sorted({int(t) for t in tiles[np.any(r > tau_local, axis=0)]})
        raise AssertionError("%s: local error %.3g x scale > %.3g at channel %d, sample %d (tile %d): y %.9g, float64 %.9g, "
                             "scale %.3g; %d tiles over the bound: %s" % (
                                 label, worst, tau_local, c, n0 + i, (n0 + i) // B, y[c, i], y64[c, i], scale[c, i],
                                 len(bad), bad[:12]))
    assert g <= tau_global, "%s: global relative RMS %.3g > %.3g" % (label, g, tau_global)
    return worst, g


# ------------------------------------------------------------------------------------------------ structured inputs
def white_dry(rng, N):
    """(a) the baseline dry signal."""
    return so.synth_dry(rng, N)


def graded_dry(rng, N, silent=0.2):
    """(b) white noise with every 4096-sample grid block scaled by its own power of two in 2^-6 .. 2^6, about `silent`
    of the blocks silent (the first block never, so the stem is not trivially zero): a wrong dry window, a wrong X or
    a wrong history before a block brings in a block of another level."""
    x = so.synth_dry(rng, N).astype(np.float64)
    nb = -(-N // B)
    g = 2.0 ** rng.integers(-6, 7, nb)
    g[1:][rng.random(nb - 1) < silent] = 0.0
    return (x * np.repeat(g, B)[:N]).astype(np.float32)


def impulse_dry(N, period=997, phase=3):
    """(d) an impulse train: unit impulses of alternating sign and levels 1, 1/2, 1/4 every `period` samples (prime to
    4096, so the impulses visit every offset inside a block)."""
    x = np.zeros(N, np.float32)
    k = np.arange(phase % max(N, 1), N, period)
    x[k] = np.float32(1.0) * np.where(np.arange(k.size) % 2, -1.0, 1.0) * 2.0 ** -(np.arange(k.size) % 3)
    return x


def delay_taps(L):
    """The delays of delay_rirs: 0, 1, 4095, 4096, 4097 and L - 1 where they fit."""
    return sorted({d for d in (0, 1, B - 1, B, B + 1, L - 1) if 0 <= d < L})


def delay_rirs(rng, P, C, L):
    """(c) pure-delay RIRs h[p, c, k] = g_pc delta[k - d_pc]: the gains distinct per position and channel (in
    [0.5, 1], either sign), the delays cycling through delay_taps(L) so that partition starts and ends, the block
    length and the last tap all occur.  A wrong position, channel, partition offset or sample shift moves a whole
    scaled copy of the dry signal.  Returns (h, delays (P, C))."""
    taps = delay_taps(L)
    h = np.zeros((P, C, L), np.float32)
    g = 0.5 + 0.5 * (rng.permutation(P * C) + 1) / (P * C)
    g = (g * rng.choice([-1.0, 1.0], P * C)).reshape(P, C)
    d = np.zeros((P, C), np.int64)
    off = int(rng.integers(0, len(taps)))
    for p in range(P):
        for c in range(C):
            d[p, c] = taps[(off + p * C + c) % len(taps)]
            h[p, c, d[p, c]] = g[p, c]
    return h, d


def dry_signal(kind, rng, N):
    """dry input of kind 'white' (a), 'graded' (b) or 'impulse' (d)."""
    if kind == "white":
        return white_dry(rng, N)
    if kind == "graded":
        return graded_dry(rng, N)
    if kind == "impulse":
        return impulse_dry(N)
    raise ValueError(kind)


def rir_set(kind, rng, P, C, L):
    """RIRs of kind 'synth' (decaying noise, so.synth_rirs) or 'delay' (c)."""
    if kind == "synth":
        return so.synth_rirs(rng, P, C, L)
    if kind == "delay":
        return delay_rirs(rng, P, C, L)[0]
    raise ValueError(kind)
