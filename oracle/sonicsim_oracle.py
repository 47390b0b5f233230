"""CPU oracle for the SonicSim moving-source render hot path.

TEST INFRASTRUCTURE.  Only tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs may import this file.  The product
(sonicsim_b200/) never does: it fails loudly when the CUDA library is missing.

Every function restates one reference function (file:line relative to
/root/reference/) with the same third-party calls the reference makes, so that
its results AND its CPU cost are the reference's:

  setup_dynamic_interp      SonicSim-SonicSet/SonicSim_moving.py:15-45
  convolve_fixed_receiver   SonicSim-SonicSet/SonicSim_moving.py:47-61   (scipy.signal.fftconvolve)
  convolve_moving_receiver  SonicSim-SonicSet/SonicSim_moving.py:63-96   (scipy.signal.oaconvolve + gather + lerp)
  interpolate_moving_audio  SonicSim-SonicSet/SonicSim_moving.py:98-125
  fft_conv                  SonicSim-SonicSet/SonicSim_audio.py:17-47    (torch.fft)
  lufs_norm / get_lufs_norm_audio  SonicSim-SonicSet/SonicSim_audio.py:68-86 (pyloudnorm 0.1.1)

Pinning status
  * a1-a4, a6: PINNED against the live reference, run in the authoring container by
    oracle/make_golden.py -> tests/golden/*.npz (tests/test_oracle_golden.py), and
    re-checked live whenever /root/reference is present.
  * a5 (loudness): "parity unpinned".  pyloudnorm==0.1.1 (ss-2.0.yaml:201) is not
    vendored in the reference and not installable here (no network); `bs1770_*`
    below restate ITU-R BS.1770-4 as pyloudnorm 0.1.1 implements it, from its
    published algorithm.  Cross-check against the package when a box has it.

Third-party arithmetic: scipy.signal.{fftconvolve,oaconvolve}; reference pins
scipy==1.9.1 (ss-2.0.yaml:223), this image has scipy 1.18.1.  Linear convolution
is version independent up to fp32 rounding (rel. RMS ~3e-7, SURVEY section 6).
"""
import math

import numpy as np
from scipy import signal


# --------------------------------------------------------------------------- a1
def setup_dynamic_interp(receiver_position, total_samples):
    """SonicSim_moving.py:15-45.  Same NumPy global-RNG call sequence as the reference
    (`np.random.choice(S, |err|)`, :38), so seeding np.random before the call gives
    bit-identical (interp_index int64, interp_weight float32)."""
    receiver_position = np.asarray(receiver_position)
    distance = np.linalg.norm(np.diff(receiver_position, axis=0), axis=1)            # :32
    speed_per_sample = distance.sum() / total_samples                               # :33
    samples_per_interval = np.round(distance / speed_per_sample).astype(int)        # :34
    error = total_samples - samples_per_interval.sum()                              # :37
    for i in np.random.choice(len(samples_per_interval), abs(error)):               # :38
        samples_per_interval[i] += np.sign(error)                                   # :39
    interp_index = np.repeat(np.arange(len(distance)), samples_per_interval)        # :42
    interp_weight = np.concatenate(
        [np.linspace(0, 1, num, endpoint=False) for num in samples_per_interval])   # :43
    return interp_index, interp_weight.astype(np.float32)


def samples_per_interval_from_index(interp_index, num_segments):
    """Compact form of (idx, w) produced by setup_dynamic_interp: the per-segment sample
    counts (np.repeat counts of :42).  Test helper."""
    return np.bincount(np.asarray(interp_index), minlength=num_segments).astype(np.int64)


# --------------------------------------------------------------------------- a4
def convolve_fixed_receiver(source_audio, rirs):
    """SonicSim_moving.py:47-61: full FFT convolution, truncated to the dry length."""
    source_audio = np.asarray(source_audio)
    rirs = np.asarray(rirs)
    return signal.fftconvolve(source_audio.reshape(1, -1), rirs, mode="full")[:, : source_audio.shape[-1]]


# --------------------------------------------------------------------------- a2
def convolve_moving_receiver(source_audio, rirs, interp_index, interp_weight):
    """SonicSim_moving.py:63-96: dry (*) every position's RIR, gather adjacent positions, lerp."""
    num_channels = rirs.shape[1]
    audio_len = source_audio.shape[0]
    convolved = signal.oaconvolve(source_audio[None, None, :], rirs, axes=-1)[..., :audio_len]   # :86
    ch = np.arange(num_channels)[:, None]
    n = np.arange(audio_len)
    start_audio = convolved[interp_index, ch, n]                                             # :89
    end_audio = convolved[interp_index + 1, ch, n]                                           # :90
    w = interp_weight[None, :]                                                               # :91
    return (1 - w) * start_audio + w * end_audio                                             # :94


def interpolate_moving_audio(source1_audio, ir1_list, receiver_position):
    """SonicSim_moving.py:98-125 on NumPy arrays: (1,N), (P,1,C,L), (P,3) -> (C,N)."""
    source1_audio = np.asarray(source1_audio)
    audio_len = source1_audio.shape[-1]
    idx, w = setup_dynamic_interp(np.array(receiver_position), audio_len)            # :119
    out = convolve_moving_receiver(source1_audio[0], np.asarray(ir1_list).squeeze(1), idx, w)  # :122
    return out[..., :audio_len]


def convolve_moving_exact_f64(source_audio, rirs, interp_index, interp_weight):
    """float64 ground truth in the segment-local form (SURVEY 3.2):
        y[c,n] = (1-w[n]) (x*h[idx[n],c])[n] + w[n] (x*h[idx[n]+1,c])[n]
    evaluated only for the positions a sample needs.  Independent of oaconvolve's blocking."""
    x = np.asarray(source_audio, dtype=np.float64)
    h = np.asarray(rirs, dtype=np.float64)
    idx = np.asarray(interp_index).astype(np.int64)
    w = np.asarray(interp_weight, dtype=np.float64)
    n_pos, n_ch, _ = h.shape
    out = np.zeros((n_ch, x.shape[0]), dtype=np.float64)
    for p in range(n_pos):
        sel0 = idx == p
        sel1 = (idx + 1) == p
        if not (sel0.any() or sel1.any()):
            continue
        conv = signal.fftconvolve(x[None, :], h[p], mode="full")[:, : x.shape[0]]
        out[:, sel0] += (1.0 - w[sel0])[None, :] * conv[:, sel0]
        out[:, sel1] += w[sel1][None, :] * conv[:, sel1]
    return out


# --------------------------------------------------------------------------- a6
def fft_conv(sig, kernel):
    """SonicSim_audio.py:17-47 (torch.fft): zero-pad both to N+L-1, rfft * rfft -> irfft.
    No truncation.  Takes / returns torch tensors like the reference."""
    import torch
    import torch.nn.functional as F
    padded_signal = F.pad(sig.reshape(-1), (0, kernel.size(-1) - 1))
    padded_kernel = F.pad(kernel.reshape(-1), (0, sig.size(-1) - 1))
    out_fr = torch.fft.rfftn(padded_signal, dim=-1) * torch.fft.rfftn(padded_kernel, dim=-1)
    return torch.fft.irfftn(out_fr, dim=-1)


# --------------------------------------------------------------------------- a5
# pyloudnorm 0.1.1 restatement ("parity unpinned", see module docstring).
_BS1770_G = [1.0, 1.0, 1.0, 1.41, 1.41]        # pyloudnorm/meter.py channel gains
# The library's extension to 6-8 channels (mic arrays; include/sonicsim_b200.h ss_loudness_dev): weight 1 beyond
# pyloudnorm's five.  Off by default, where more than five channels raise as in pyloudnorm.
_BS1770_G8 = _BS1770_G + [1.0, 1.0, 1.0]


def bs1770_k_weighting(rate):
    """pyloudnorm 0.1.1 Meter 'K-weighting': IIRfilter(4.0, 1/sqrt(2), 1500, rate, 'high_shelf')
    then IIRfilter(0.0, 0.5, 38.0, rate, 'high_pass'); RBJ-cookbook coefficients evaluated at the
    actual sample rate.  Returns [(b, a), (b, a)], each normalised by a0."""
    out = []
    for (G, Q, fc, kind) in ((4.0, 1.0 / np.sqrt(2.0), 1500.0, "high_shelf"),
                             (0.0, 0.5, 38.0, "high_pass")):
        A = 10.0 ** (G / 40.0)
        w0 = 2.0 * np.pi * (fc / rate)
        alpha = np.sin(w0) / (2.0 * Q)
        if kind == "high_shelf":
            b0 = A * ((A + 1) + (A - 1) * np.cos(w0) + 2 * np.sqrt(A) * alpha)
            b1 = -2 * A * ((A - 1) + (A + 1) * np.cos(w0))
            b2 = A * ((A + 1) + (A - 1) * np.cos(w0) - 2 * np.sqrt(A) * alpha)
            a0 = (A + 1) - (A - 1) * np.cos(w0) + 2 * np.sqrt(A) * alpha
            a1 = 2 * ((A - 1) - (A + 1) * np.cos(w0))
            a2 = (A + 1) - (A - 1) * np.cos(w0) - 2 * np.sqrt(A) * alpha
        else:
            b0 = (1 + np.cos(w0)) / 2
            b1 = -(1 + np.cos(w0))
            b2 = (1 + np.cos(w0)) / 2
            a0 = 1 + alpha
            a1 = -2 * np.cos(w0)
            a2 = 1 - alpha
        out.append((np.array([b0, b1, b2]) / a0, np.array([a0, a1, a2]) / a0))
    return out


def bs1770_block_bounds(num_samples, rate, block_size):
    """Gating-block sample bounds exactly as pyloudnorm computes them (float expressions
    truncated with int()), 75 % overlap.  Returns (l, u) int64 arrays of length numBlocks."""
    T_g = block_size
    step = 1.0 - 0.75
    T = num_samples / rate
    num_blocks = int(np.round(((T - T_g) / (T_g * step))) + 1)
    lo = np.array([int(T_g * (j * step) * rate) for j in range(num_blocks)], dtype=np.int64)
    hi = np.array([int(T_g * (j * step + 1) * rate) for j in range(num_blocks)], dtype=np.int64)
    return lo, hi


def _bs1770_gating(data, rate, block_size, up_to_8_channels):
    """The steps of integrated_loudness: (block loudness l_j, relative gate gamma_r, integrated loudness)."""
    data = np.asarray(data)
    if not np.issubdtype(data.dtype, np.floating):
        raise ValueError("Data must be floating point.")
    max_ch = 8 if up_to_8_channels else 5
    if data.ndim == 2 and data.shape[1] > max_ch:
        raise ValueError("Audio must have five channels or less." if max_ch == 5 else
                         "Audio must have eight channels or less.")
    if data.shape[0] < block_size * rate:
        raise ValueError("Audio must have length greater than the block size.")
    x = data.copy()
    if x.ndim == 1:
        x = x.reshape(-1, 1)
    n_samp, n_ch = x.shape
    for (b, a) in bs1770_k_weighting(rate):
        for ch in range(n_ch):
            x[:, ch] = signal.lfilter(b, a, x[:, ch])       # float64 filter, stored back in x.dtype
    lo, hi = bs1770_block_bounds(n_samp, rate, block_size)
    T_g = block_size
    nb = len(lo)
    z = np.zeros((n_ch, nb))
    for i in range(n_ch):
        for j in range(nb):
            z[i, j] = (1.0 / (T_g * rate)) * np.sum(np.square(x[lo[j]:hi[j], i]))
    G = _BS1770_G8 if up_to_8_channels else _BS1770_G
    with np.errstate(divide="ignore", invalid="ignore"):
        l = [-0.691 + 10.0 * np.log10(np.sum([G[i] * z[i, j] for i in range(n_ch)])) for j in range(nb)]
        J_g = [j for j, l_j in enumerate(l) if l_j >= -70.0]
        z_avg = [np.mean([z[i, j] for j in J_g]) for i in range(n_ch)]
        gamma_r = -0.691 + 10.0 * np.log10(np.sum([G[i] * z_avg[i] for i in range(n_ch)])) - 10.0
        J_g = [j for j, l_j in enumerate(l) if (l_j > gamma_r and l_j > -70.0)]
        z_avg = np.nan_to_num(np.array([np.mean([z[i, j] for j in J_g]) for i in range(n_ch)]))
        lufs = -0.691 + 10.0 * np.log10(np.sum([G[i] * z_avg[i] for i in range(n_ch)]))
    return np.array(l, dtype=np.float64), float(gamma_r), float(lufs)


def bs1770_integrated_loudness(data, rate, block_size=0.400, up_to_8_channels=False):
    """pyloudnorm 0.1.1 Meter(rate, block_size=...).integrated_loudness(data), data (N,C) or (N,).
    `up_to_8_channels`: accept 6-8 channels with weight 1 for channels 5-7 (the library's extension)."""
    return _bs1770_gating(data, rate, block_size, up_to_8_channels)[2]


def bs1770_block_loudness(data, rate, block_size=0.400, up_to_8_channels=False):
    """(loudness of every gating block, relative gate) of integrated_loudness, for tests that must keep their
    signals away from the two gates."""
    l, gamma_r, _ = _bs1770_gating(data, rate, block_size, up_to_8_channels)
    return l, gamma_r


def lufs_norm(data, sr, norm=-6, up_to_8_channels=False):
    """SonicSim_audio.py:68-81.  Output kept in the input dtype (float32), which is what the
    reference's pinned numpy 1.23.5 produces for `np.float64 scalar * float32 array`."""
    data = np.asarray(data)
    block_size = 0.4 if len(data) / sr >= 0.4 else len(data) / sr                   # :69
    loudness = bs1770_integrated_loudness(data, sr, block_size, up_to_8_channels)   # :71-72
    if math.isinf(loudness):                                                        # :73
        loudness = -40
    gain_lin = np.power(10.0, (norm - loudness) / 20.0)                             # pyln.normalize.loudness
    norm_data = (gain_lin * data).astype(data.dtype)
    n, d = np.sum(np.array(norm_data)), np.sum(np.array(data))                      # :78
    gain = n / d if d else 0.0                                                      # :79
    return norm_data, gain


def get_lufs_norm_audio(audio, sr=16000, lufs=-6):
    """SonicSim_audio.py:83-86: target ~ U(lufs-2, lufs+2) from the global NumPy RNG."""
    class_lufs = np.random.uniform(lufs - 2, lufs + 2)                              # :84
    return lufs_norm(data=audio, sr=sr, norm=class_lufs)


# --------------------------------------------------------------------------- f1: mixture assembly
def compute_mch_rms_dB(mch_wav):
    """separation/look2hear/datas/movingdatamodule.py:29-32 (torch tensor in)."""
    import torch
    mean_square = max(1e-20, torch.mean(mch_wav ** 2))
    return 10 * np.log10(mean_square)


def mix_stems(speaker_wav, noise_wav, sirs, snr):
    """separation/look2hear/datas/movingdatamodule.py:105-124 with the random SIRs / SNR passed in
    (the reference draws them with torch.Tensor(n).uniform_).  speaker_wav (S, ..., T), noise_wav
    (M, ..., T) torch float32; returns (mix_wav, scaled speaker_wav)."""
    import torch
    speaker_wav = speaker_wav.clone()
    num_spks = speaker_wav.shape[0]
    target_refch_energy = compute_mch_rms_dB(speaker_wav[0])                       # :107
    for i in range(num_spks - 1):                                                  # :109
        sir = sirs[i]
        intf_refch_energy = compute_mch_rms_dB(speaker_wav[i + 1])
        gain = min(target_refch_energy - intf_refch_energy - sir, 40)              # :112
        speaker_wav[i + 1] *= 10. ** (gain / 20.)                                  # :113
    all_speech = torch.sum(speaker_wav, dim=0)                                     # :115
    all_noise = torch.sum(noise_wav, dim=0)                                        # :116
    target_refch_energy = compute_mch_rms_dB(all_speech)                           # :118
    noise_refch_energy = compute_mch_rms_dB(all_noise)                             # :120
    gain = min(target_refch_energy - noise_refch_energy - snr, 40)                 # :121
    all_noise = all_noise * 10. ** (float(np.asarray(gain).reshape(-1)[0]) / 20.)  # :122
    return all_speech + all_noise, speaker_wav                                     # :124


def overlap_audio(waveform, sample_rate, delay=6):
    """enhancement/look2hear/datas/movingdatamodule.py:34-48: y[n] = (x[n-D] + x[n+D]) + x[n] with zeros outside
    [0, T), D = int(delay * sample_rate); waveform (rows, T) float32 ndarray."""
    x = np.asarray(waveform, dtype=np.float32)
    T = x.shape[1]
    D = int(delay * sample_rate)                                                   # :35
    fwd = np.zeros_like(x)
    bwd = np.zeros_like(x)
    if D < T:
        fwd[:, D:] = x[:, : T - D]                                                 # :38,42
        bwd[:, : T - D] = x[:, D:]                                                 # :39,43
    return (fwd + bwd) + x                                                         # :46


def find_overlap_region(data, min_overlap=2, max_overlap=3, max_duration=None, sample_rate=None, rand=None):
    """:50-75: rejection sampling of [start, end] (inclusive `random.randint` draws) until the number of utterance
    boundaries inside it is in [min_overlap, max_overlap]; `max_duration` is (as in the reference) a MINIMUM."""
    import random as _random
    rand = rand or _random
    pts = [p for src in data.values() if "start_end_points" in src for p in src["start_end_points"]]   # :51-54
    lo = min(p[0] for p in pts)
    hi = max(p[1] for p in pts)
    while True:
        a = rand.randint(lo, hi)                                                   # :61
        b = rand.randint(a, hi)                                                    # :62
        if max_duration is not None and sample_rate is not None and (b - a) / sample_rate < max_duration:
            continue                                                               # :64-67
        n = sum(a <= p[0] <= b or a <= p[1] <= b for p in pts)                     # :69-72
        if min_overlap <= n <= max_overlap:
            return a, b


def mix_noisy(speaker_wavs, noise_wav, snr, sample_rate, delay=6):
    """:235-257 (noisy single-speaker mixture of the enhancement dataloader): summed noise stems, overlap_audio over
    the flattened signal, SNR gain (clamped at +40 dB) against the speaker stem, sum.  torch float32 in/out."""
    import torch
    all_noise = torch.sum(noise_wav, dim=0)                                        # :239
    shape = all_noise.shape
    all_noise = torch.from_numpy(overlap_audio(all_noise.reshape(1, -1).numpy(), sample_rate, delay)).reshape(shape)
    gain = min(compute_mch_rms_dB(speaker_wavs) - compute_mch_rms_dB(all_noise) - snr, 40)    # :243-246
    all_noise = all_noise * 10. ** (float(np.asarray(gain).reshape(-1)[0]) / 20.)              # :247
    return speaker_wavs + all_noise                                                # :257


# ------------------------------------------------------------------- synthetic inputs
def synth_rirs(rng, P, C, L, sr=16000, t60=0.5):
    """SURVEY 8(d): decaying Gaussian noise, small random per-position delay, divided by the
    global abs-max (as generate_rir_combination does, SonicSim_audio.py:398)."""
    t = np.arange(L) / sr
    env = np.exp(-6.9 * t / t60)
    h = rng.standard_normal((P, C, L)) * env
    for p in range(P):
        d = min(int(rng.integers(0, 65)), L // 2)
        if d:
            h[p] = np.concatenate([np.zeros((C, d)), h[p, :, : L - d]], axis=1)
    h /= np.abs(h).max()
    return h.astype(np.float32)


def synth_dry(rng, N):
    return (rng.standard_normal(N) * 0.1).astype(np.float32)


def synth_path(rng, P):
    return np.cumsum(rng.standard_normal((P, 3)), axis=0)


def rel_rms(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    den = np.sqrt(np.mean(b * b))
    return float(np.sqrt(np.mean((a - b) ** 2)) / den) if den > 0 else float(np.sqrt(np.mean((a - b) ** 2)))
