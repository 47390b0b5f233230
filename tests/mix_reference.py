"""Plain restatements of the mixture, overlap and dry-assembly kernels (csrc/ss_mix.cu, csrc/ss_dry.cu) that the CPU and
GPU tests compare them against: float64 gains and resampling, and the exact float32 composition of a mixture once its
gains are fixed.  Import-only."""
import math

import numpy as np

F32 = np.float32


def _rms_db(x):
    """compute_mch_rms_dB (movingdatamodule.py:29-32) in float64 over the float32 values of `x`."""
    v = np.asarray(x, np.float64).reshape(-1)
    return 10.0 * math.log10(max(1e-20, float(np.dot(v, v)) / v.size))


def _rows(a):
    a = np.asarray(a, F32)
    return a.reshape(a.shape[0], -1)


def overlap_exact(x, D):
    """overlap_audio with an integer shift D in samples: y[r][n] = fl(fl(x[r][n-D] + x[r][n+D]) + x[r][n]), zeros
    outside [0, T).  x (rows, T) float32."""
    x = np.asarray(x, F32)
    T = x.shape[-1]
    f = np.zeros_like(x)
    b = np.zeros_like(x)
    if D < T:
        f[..., D:] = x[..., :T - D]
        b[..., :T - D] = x[..., D:]
    return (f + b) + x


def noise_signal(noise, delay):
    """The noise rows summed in m order from 0 in float32, then (delay > 0) overlap_exact over the flattened sum."""
    n = _rows(noise)
    acc = np.zeros(n.shape[1], F32)
    for m in range(n.shape[0]):
        acc = acc + n[m]
    return overlap_exact(acc[None], int(delay))[0] if delay > 0 else acc


def compose_mix(spk, noise, g_f32, gn_f32, delay=0):
    """The mixture once the float32 gains are fixed: speakers_out[s] = fl(spk[s] * g_s); speech is the sum of
    speakers_out in s order from 0; mix = fl(speech + fl(noise_signal * gn)).  Returns (mix (E,), speakers_out (S, E))."""
    s = _rows(spk)
    out = s * np.asarray(g_f32, F32).reshape(-1, 1)
    speech = np.zeros(s.shape[1], F32)
    for r in out:
        speech = speech + r
    return speech + noise_signal(noise, delay) * F32(gn_f32), out


def mix_gains_f64(spk, noise, sirs, snr, delay=0):
    """The float64 gains of the dataloader's formulas (movingdatamodule.py:105-124): g_0 = 1, g_s = 10^(min(E_0 - E_s -
    sir_s, 40) / 20), and the noise gain 10^(min(E_speech - E_noise - snr, 40) / 20), where E is compute_mch_rms_dB
    and the speech is composed with the float32 roundings of the g_s as the write pass composes it.
    Returns (g (S,) float64, gn float64)."""
    s = _rows(spk)
    target = _rms_db(s[0])
    g = [1.0]
    for i in range(1, s.shape[0]):
        g.append(10.0 ** (min(target - _rms_db(s[i]) - float(F32(sirs[i - 1])), 40.0) / 20.0))
    g = np.array(g)
    speech = compose_mix(s, np.zeros((1, s.shape[1]), F32), g.astype(F32), 0.0)[0]
    gn = 10.0 ** (min(_rms_db(speech) - _rms_db(noise_signal(noise, delay)) - float(F32(snr)), 40.0) / 20.0)
    return g, gn


def f32_neighbours(g64, k=3):
    """The float32 values within k ulps of fl32(g64), in increasing order."""
    c = [F32(g64)]
    for _ in range(k):
        c.insert(0, np.nextafter(c[0], F32(-np.inf)))
        c.append(np.nextafter(c[-1], F32(np.inf)))
    return c


def ulps_f32(a, g64):
    """Number of float32 steps between float32 `a` and fl32(g64) (both positive)."""
    return abs(int(np.array(a, F32).view(np.int32)) - int(np.array(g64, F32).view(np.int32)))


def assert_clear_of_f32_midpoint(g64, margin=1e-9):
    """`g64` is not within a relative `margin` of a point halfway between two float32 values, so any float64 result
    close to it rounds to the same float32 and a bit-exactness claim cannot turn on a near-tie."""
    f = F32(g64)
    for nb in (np.nextafter(f, F32(-np.inf)), np.nextafter(f, F32(np.inf))):
        mid = (float(f) + float(nb)) / 2.0
        assert abs(g64 - mid) > margin * abs(g64), (g64, mid)


def resample_kernel(orig, new):
    """torchaudio.transforms.Resample(orig, new)'s own float32 filter bank as (K (new_g, taps) float32, orig_g, new_g,
    width), the rates divided by their gcd."""
    import torchaudio
    rs = torchaudio.transforms.Resample(orig_freq=orig, new_freq=new)
    g = math.gcd(int(orig), int(new))
    return rs.kernel[:, 0, :].numpy().astype(F32), int(orig) // g, int(new) // g, int(rs.width)


RESAMPLE_PAIRS = [(8000, 16000), (11025, 16000), (22050, 16000), (24000, 16000), (32000, 16000), (44100, 16000),
                  (48000, 16000), (16000, 48000), (44100, 48000)]


def clip_lengths(orig, new):
    """1, 2, width, taps - 1, taps, taps + 1, orig +- 1 (rates divided by their gcd) and about 10 s."""
    K, o, n, width = resample_kernel(orig, new)
    taps = K.shape[1]
    return sorted({v for v in (1, 2, width, taps - 1, taps, taps + 1, o - 1, o + 1, 10 * orig + 7) if v >= 1})


def _frames(x, orig, new):
    K, o, n, width = resample_kernel(orig, new)
    x = np.asarray(x, np.float64).reshape(-1)
    taps = K.shape[1]
    xpad = np.concatenate([np.zeros(width), x, np.zeros(width + o)])
    fr = np.lib.stride_tricks.sliding_window_view(xpad, taps)[::o]
    return fr, K.astype(np.float64), -(-n * x.size // o)


def resample_f64(x, orig, new):
    """torchaudio.transforms.Resample(orig, new)(x) in float64 with the same filter bank:
    y[j * new + p] = sum_k K[p][k] * xpad[j * orig + k], xpad = `width` zeros, x, `width + orig` zeros, truncated to
    ceil(new * len / orig) (rates divided by their gcd)."""
    fr, K, n_out = _frames(x, orig, new)
    return (fr @ K.T).reshape(-1)[:n_out]


def resample_abs_bound(x, orig, new):
    """sum_k |K[p][k] * xpad[j * orig + k]| for every output sample of resample_f64: the scale of the rounding error of
    any order of the sum."""
    fr, K, n_out = _frames(x, orig, new)
    return (np.abs(fr) @ np.abs(K).T).reshape(-1)[:n_out]


def max_rel(y, y64):
    """max |y - y64| / max |y64| (0 for an all-zero y64 matched exactly)."""
    y64 = np.asarray(y64, np.float64)
    err = float(np.max(np.abs(np.asarray(y, np.float64) - y64))) if y64.size else 0.0
    den = float(np.max(np.abs(y64))) if y64.size else 0.0
    return err / den if den > 0 else err
