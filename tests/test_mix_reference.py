"""The references of tests/mix_reference.py against the unmodified reference: compose_mix reproduces the golden
mixtures bit for bit from the reference's own float32 gains, mix_gains_f64 lies within 3 ulps of those gains,
overlap_exact reproduces overlap_audio bit for bit, and resample_f64 matches torchaudio's Resample."""
import numpy as np
import pytest
import torch

from mix_reference import (F32, RESAMPLE_PAIRS, clip_lengths, compose_mix, mix_gains_f64, overlap_exact,
                           resample_abs_bound, resample_f64, ulps_f32)
from oracle import sonicsim_oracle as so


def reference_gains_f32(spk, noise, sirs, snr, delay_s=None, sr=None):
    """The gains the reference computes (movingdatamodule.py:105-124, enhancement :243-247), through the oracle's
    compute_mch_rms_dB, which tests/test_mix.py pins to the reference's lines: float32 tensors for the speakers, a
    Python float multiplier for the noise.  Returns (g (S,) float32, gn float32, D)."""
    spk_t = torch.from_numpy(spk)
    g = [F32(1.0)]
    t = so.compute_mch_rms_dB(spk_t[0])
    for i in range(spk.shape[0] - 1):
        gain = min(t - so.compute_mch_rms_dB(spk_t[i + 1]) - sirs[i], 40)
        g.append(F32(float(10. ** (gain / 20.))))
    scaled = spk_t.clone()
    for i in range(1, spk.shape[0]):
        scaled[i] *= torch.tensor(g[i])
    all_noise = torch.sum(torch.from_numpy(noise), dim=0)
    D = 0
    if delay_s is not None:
        D = int(delay_s * sr)
        all_noise = torch.from_numpy(so.overlap_audio(all_noise.reshape(1, -1).numpy(), sr, delay_s)).reshape(all_noise.shape)
    gain = min(so.compute_mch_rms_dB(torch.sum(scaled, dim=0)) - so.compute_mch_rms_dB(all_noise) - snr, 40)
    return np.array(g, F32), F32(10. ** (float(np.asarray(gain).reshape(-1)[0]) / 20.)), D


def _golden_cases(golden):
    g = golden("mix_stems")
    for k in range(int(g["n_cases"])):
        yield (f"stems{k}", g[f"spk{k}"], g[f"noise{k}"], g[f"sirs{k}"], g[f"snr{k}"], None, None,
               g[f"mix{k}"], g[f"spk_out{k}"])
    g = golden("mix_noisy")
    for k in range(int(g["n_mn"])):
        yield (f"noisy{k}", g[f"mn_spk{k}"][None], g[f"mn_noise{k}"], [], g[f"mn_snr{k}"], 6, int(g[f"mn_sr{k}"]),
               g[f"mn_mix{k}"], None)


def test_compose_mix_reproduces_golden_bit_exact(golden):
    n = 0
    for name, spk, noise, sirs, snr, delay_s, sr, want_mix, want_spk in _golden_cases(golden):
        g, gn, D = reference_gains_f32(spk, noise, sirs, snr, delay_s, sr)
        mix, out = compose_mix(spk, noise, g, gn, D)
        assert np.array_equal(mix, want_mix.reshape(-1)), name
        if want_spk is not None:
            assert np.array_equal(out, want_spk.reshape(want_spk.shape[0], -1)), name
        n += 1
    assert n == 6


def test_mix_gains_f64_within_3_ulps_of_reference(golden):
    for name, spk, noise, sirs, snr, delay_s, sr, _, _ in _golden_cases(golden):
        g, gn, D = reference_gains_f32(spk, noise, sirs, snr, delay_s, sr)
        g64, gn64 = mix_gains_f64(spk.reshape(spk.shape[0], -1), noise.reshape(noise.shape[0], -1), sirs,
                                  float(np.asarray(snr).reshape(-1)[0]), D)
        assert g64[0] == 1.0
        for s in range(1, len(g)):
            assert ulps_f32(g[s], g64[s]) <= 3, (name, s, g[s], g64[s])
        assert ulps_f32(gn, gn64) <= 3, (name, gn, gn64)


def test_compose_mix_edges():
    """delay 0 is no overlap; every shift at or past the signal's end leaves only the centre term; zeros stay zeros."""
    rng = np.random.default_rng(5)
    n = rng.standard_normal((3, 10)).astype(F32)
    s = rng.standard_normal((2, 10)).astype(F32)
    for D in (10, 11, 2 ** 40):
        assert np.array_equal(overlap_exact(n, D), n)
    assert np.array_equal(compose_mix(s, n, [1.0, 0.5], 2.0, 0)[0],
                          (s[0] + s[1] * F32(0.5)) + ((n[0] + n[1]) + n[2]) * F32(2.0))
    mix, out = compose_mix(np.zeros((2, 7), F32), np.zeros((1, 7), F32), [1.0, 100.0], 100.0, 3)
    assert not mix.any() and not out.any()


def test_overlap_exact_matches_golden(golden):
    g = golden("mix_noisy")
    for k in range(int(g["n_ov"])):
        D = int(float(g[f"ov_delay{k}"]) * int(g[f"ov_sr{k}"]))
        assert np.array_equal(overlap_exact(g[f"ov_x{k}"], D), g[f"ov_y{k}"])


@pytest.mark.parametrize("orig,new", RESAMPLE_PAIRS)
def test_resample_f64_matches_torchaudio(orig, new):
    import torchaudio
    rs = torchaudio.transforms.Resample(orig_freq=orig, new_freq=new)
    rng = np.random.default_rng(orig + new)
    for L in clip_lengths(orig, new):
        x = (rng.standard_normal(L) * 0.1).astype(F32)
        want = rs(torch.from_numpy(x)[None])[0].numpy().astype(np.float64)
        got = resample_f64(x, orig, new)
        assert got.shape == want.shape, (L, got.shape, want.shape)
        err = np.max(np.abs(got - want)) / np.max(np.abs(want))
        assert err <= 1e-6, (orig, new, L, err)
        b = resample_abs_bound(x, orig, new)
        assert b.shape == got.shape and np.all(np.abs(got) <= b * (1 + 1e-12))
