"""Plain restatements of the mixture, overlap and dry-assembly kernels (csrc/ss_mix.cu, csrc/ss_dry.cu) that the CPU and
GPU tests compare them against: float64 gains and resampling, and the exact float32 composition of a mixture once its
gains are fixed; and the guarded device buffers, mixture items and checkers the GPU tests run them through.  Import-only."""
import math

import numpy as np
import torch

from gpu_plumbing import _stream, renderer

F32 = np.float32
NAN = float("nan")


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

PAD = 37

SENT = 1234.5

GUARD = 64

MAX_ULPS = [0]          # largest gain error seen, in float32 steps from fl32(g64)


def fold(a):
    """Channel mean of a (C, T) stem as SS_MIX_MONO computes it: float32 sum in channel order, then / C."""
    a = np.asarray(a, F32)
    acc = a[0].copy()
    for c in range(1, a.shape[0]):
        acc = acc + a[c]
    return acc / F32(a.shape[0])


class Out:
    """A (rows, n) output inside a NaN-filled device buffer with sentinels on both sides."""

    def __init__(self, rows, n):
        self.rows, self.n = rows, n
        self.buf = torch.full((rows * n + 2 * PAD,), float("nan"), device="cuda")
        self.buf[:PAD] = SENT
        self.buf[-PAD:] = SENT

    def ptr(self):
        return self.buf.data_ptr() + 4 * PAD

    def view(self, *shape):
        return self.buf[PAD:PAD + self.rows * self.n].view(*(shape or (self.rows, self.n)))

    def reset(self):
        self.buf[PAD:-PAD].fill_(float("nan"))

    def get(self, snap=None):
        """The output of a snapshot of the buffer (default: the buffer now) as (rows, n), sentinels and fill checked."""
        s = self.buf if snap is None else snap
        a = s.cpu().numpy() if isinstance(s, torch.Tensor) else s
        assert np.all(a[:PAD] == SENT) and np.all(a[-PAD:] == SENT), "sentinel overwritten"
        v = a[PAD:-PAD].reshape(self.rows, self.n)
        assert not np.isnan(v).any(), "output not written"
        return v


def check_mixture(spk, noi, sirs, snr, mix, out, rms, label=""):
    """A plan mixture against mix_reference: speaker 0 unscaled, every other speaker gain and the noise gain a float32
    within 3 ulps of the float64 gain, speakers_out and mix bit for bit compose_mix with those gains, rms_db within
    1e-6 dB of the float64 RMS, or within half a float32 step of it where that is larger (beyond 32 dB from 0 a float32
    step is 3.8e-6 dB, and rms_db is the float64 value rounded to float32).  spk (S, E), noi (M, E) are the stems the
    mixture must have read."""
    S = spk.shape[0]
    g64, gn64 = mix_gains_f64(spk, noi, sirs, snr)
    assert np.array_equal(out[0], spk[0]), label
    g = [F32(1.0)]
    for s in range(1, S):
        fits = [v for v in f32_neighbours(g64[s]) if np.array_equal(out[s], spk[s] * v)]
        assert fits, (label, "speaker", s, g64[s])
        g.append(fits[0])
    fits = [v for v in f32_neighbours(gn64) if np.array_equal(mix, compose_mix(spk, noi, g, v)[0])]
    assert fits, (label, "noise gain", gn64)
    assert np.array_equal(out, compose_mix(spk, noi, g, fits[0])[1]), label
    for s in range(S):
        r64 = _rms_db(spk[s])
        tol = max(1e-6, 0.5 * float(np.spacing(F32(abs(r64)))) + 1e-12)
        assert abs(float(rms[s]) - r64) <= tol, (label, s, rms[s], r64)


class MixBuf:
    """`n` values at `off` elements past a NaN guard of GUARD elements, followed by GUARD NaNs."""

    def __init__(self, n, off=0, data=None, dtype=torch.float32):
        self.n, self.lo = int(n), GUARD + off
        self.t = torch.full((GUARD + off + self.n + GUARD,), NAN, dtype=dtype, device="cuda")
        if data is not None:
            self.t[self.lo:self.lo + self.n] = torch.from_numpy(np.ascontiguousarray(data).reshape(-1)).cuda()

    @property
    def ptr(self):
        return self.t.data_ptr() + self.lo * self.t.element_size()

    def get(self):
        return self.t[self.lo:self.lo + self.n].cpu().numpy()

    def guards_nan(self):
        a = self.t.cpu().numpy()
        return bool(np.all(np.isnan(a[:self.lo])) and np.all(np.isnan(a[self.lo + self.n:])))


class Mix:
    """One ss_mix_item over guarded buffers.  out: "null", "sep" (its own buffer) or "alias" (== speakers)."""

    def __init__(self, spk, noise, sirs, snr, delay=0, out="sep", offs=(0, 0, 0, 0)):
        from sonicsim_b200 import _lib as L
        self.spk, self.noise = np.asarray(spk, F32), np.asarray(noise, F32)
        self.S, self.E = self.spk.shape
        self.M = self.noise.shape[0]
        self.sirs = np.asarray(sirs, F32).reshape(-1)[:self.S - 1]
        self.snr, self.delay, self.mode = F32(snr), int(delay), out
        self.b_spk = MixBuf(self.S * self.E, offs[0], self.spk)
        self.b_noise = MixBuf(self.M * self.E, offs[1], self.noise)
        self.b_mix = MixBuf(self.E, offs[2])
        self.b_out = MixBuf(self.S * self.E, offs[3]) if out == "sep" else None
        self.b_sirs = MixBuf(max(self.S - 1, 1), 0, self.sirs if self.S > 1 else None)
        self.b_scr = MixBuf(int(renderer().lib.ss_mix_scratch_doubles()), 0, dtype=torch.float64)
        outp = {"null": None, "sep": self.b_out.ptr if self.b_out else None, "alias": self.b_spk.ptr}[out]
        self.item = L.SsMixItem(speakers=self.b_spk.ptr, noises=self.b_noise.ptr, sirs=self.b_sirs.ptr,
                                mix=self.b_mix.ptr, speakers_out=outp, scratch=self.b_scr.ptr, E=self.E, S=self.S,
                                M=self.M, snr=float(self.snr), noise_delay=self.delay)

    def bufs(self):
        return [b for b in (self.b_spk, self.b_noise, self.b_mix, self.b_out, self.b_sirs, self.b_scr) if b]

    def outputs(self):
        """(mix, speakers_out or None); checks the guards and that the speakers are unchanged unless aliased."""
        assert all(b.guards_nan() for b in self.bufs())
        spk = self.b_spk.get().reshape(self.S, self.E)
        if self.mode == "alias":
            return self.b_mix.get(), spk
        assert np.array_equal(spk, self.spk)
        return self.b_mix.get(), None if self.b_out is None else self.b_out.get().reshape(self.S, self.E)


def mix_dev(cases):
    R = renderer()
    arr = (type(cases[0].item) * len(cases))(*[c.item for c in cases])
    st = R.lib.ss_mix_dev(R.ctx, arr, len(cases), _stream())
    torch.cuda.synchronize()
    return st


def recover(out, x, g64):
    """The float32 gains g among +-3 ulps of fl32(g64) with out == fl(x * g) everywhere."""
    fits = [g for g in f32_neighbours(g64) if np.array_equal(out, x * g)]
    assert fits, ("no float32 gain within 3 ulps reproduces the output", g64)
    MAX_ULPS[0] = max(MAX_ULPS[0], min(ulps_f32(g, g64) for g in fits))
    return fits[0]


def check_mix(c, mix, spk_out):
    """Gains within 3 ulps of mix_gains_f64, g_0 == 1, and mix / speakers_out bit for bit compose_mix with them.
    Returns the recovered (g, gn)."""
    g64, gn64 = mix_gains_f64(c.spk, c.noise, c.sirs, c.snr, c.delay)
    assert spk_out is not None
    assert np.array_equal(spk_out[0], c.spk[0])                            # g_0 is exactly 1
    g = np.array([F32(1.0)] + [recover(spk_out[s], c.spk[s], g64[s]) for s in range(1, c.S)], F32)
    speech, out = compose_mix(c.spk, np.zeros((1, c.E), F32), g, 0.0)
    assert np.array_equal(out, spk_out)
    noise = compose_mix(np.zeros((1, c.E), F32), c.noise, [1.0], 1.0, c.delay)[0]
    fits = [gn for gn in f32_neighbours(gn64) if np.array_equal(mix, speech + noise * gn)]
    assert fits, ("mix is not the composition with any noise gain within 3 ulps", gn64)
    MAX_ULPS[0] = max(MAX_ULPS[0], min(ulps_f32(gn, gn64) for gn in fits))
    assert np.array_equal(mix, compose_mix(c.spk, c.noise, g, fits[0], c.delay)[0])
    return g, fits[0]


class DryBuf:
    """`n` floats at `off` past a NaN guard of `pad` floats, followed by `pad` NaNs."""

    def __init__(self, n, off=0, data=None, pad=64):
        self.n, self.lo = int(n), pad + off
        self.t = torch.full((pad + off + self.n + pad,), NAN, device="cuda")
        if data is not None:
            self.t[self.lo:self.lo + self.n] = torch.from_numpy(np.ascontiguousarray(data, F32).reshape(-1)).cuda()

    @property
    def ptr(self):
        return self.t.data_ptr() + 4 * self.lo

    def get(self):
        return self.t[self.lo:self.lo + self.n].cpu().numpy()

    def guards_nan(self):
        a = self.t.cpu().numpy()
        return bool(np.all(np.isnan(a[:self.lo])) and np.all(np.isnan(a[self.lo + self.n:])))

_banks = {}


def bank(orig, new):
    """(guarded (taps, new_g) filter bank, orig_g, new_g, width, taps) of Resample(orig, new); guards of `taps` floats."""
    if (orig, new) not in _banks:
        K, o, n, width = resample_kernel(orig, new)
        taps = K.shape[1]
        _banks[(orig, new)] = (DryBuf(taps * n, 0, K.T, pad=taps), o, n, width, taps)
    return _banks[(orig, new)]


class Clip:
    """One ss_dry_clip: x (channels, L) at `orig` Hz placed into a `new` Hz stream (orig == new: no resampling)."""

    def __init__(self, x, orig, new, src_start, count, dst_start, off=0):
        from sonicsim_b200 import _lib as L
        self.x, self.orig, self.new = np.asarray(x, F32), orig, new
        self.ch, self.L = self.x.shape
        self.src_start, self.count, self.dst_start = int(src_start), int(count), int(dst_start)
        kt, o, n, width, taps = (None, 1, 1, 0, 1) if orig == new else bank(orig, new)
        self.taps = taps
        self.src = DryBuf(self.ch * self.L, off, self.x, pad=max(taps, 64))
        self.c = L.SsDryClip(src=self.src.ptr, kernel_t=kt.ptr if kt else None, dst_start=self.dst_start,
                             src_start=self.src_start, count=self.count, channels=self.ch, src_len=self.L, orig=o,
                             new_rate=n, width=width, taps=taps)

    def expected(self):
        """(float64 clip, per-sample rounding bound) over [src_start, src_start + count); bound None: exact."""
        sl = slice(self.src_start, self.src_start + self.count)
        if self.orig == self.new:
            y = self.x[0] if self.ch == 1 else (self.x[0] + self.x[1]) * F32(0.5)
            return y[sl], None
        y = sum(resample_f64(r, self.orig, self.new) for r in self.x) / self.ch
        b = sum(resample_abs_bound(r, self.orig, self.new) for r in self.x) / self.ch
        # fp32 accumulation of at most `taps` fused terms per channel, one more rounding for the stereo sum
        return y[sl], (self.taps + self.ch - 1) * 2.0 ** -24 * b[sl]
