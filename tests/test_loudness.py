"""lufs_norm (SonicSim_audio.py:68-81): oracle (pyloudnorm 0.1.1 restatement, "parity unpinned")
against the kernels' per-thread code (CPU emulation) and, with -m gpu, the CUDA path."""
import numpy as np
import pytest

from oracle import sonicsim_oracle as so
from loudness_cases import (EXACT_DB, PARTITION_CASES, RATES, REFINES, assert_clear_of_gates, block_size_of,
                            n_samples_for, stems)


def test_oracle_kweighting_reference_values():
    """Pins of the restatement that do not need pyloudnorm: BS.1770's own 48 kHz coefficient table
    and the standard's -3.01 LKFS for a 0 dBFS 997 Hz sine (+3.01 for two channels)."""
    (b1, a1), (b2, a2) = so.bs1770_k_weighting(48000)
    assert np.allclose(b1, [1.53512485958697, -2.69169618940638, 1.19839281085285], atol=2e-3)
    assert np.allclose(a1, [1.0, -1.69065929318241, 0.73248077421585], atol=2e-3)
    assert np.allclose(b2, [1.0, -2.0, 1.0], atol=1.1e-2)      # RBJ form is a0-normalised: 0.995 * [1, -2, 1]
    assert np.allclose(a2, [1.0, -1.99004745483398, 0.99007225036621], atol=1e-4)
    sr = 48000
    t = np.arange(sr * 5) / sr
    sine = np.sin(2 * np.pi * 997 * t).astype(np.float32)
    assert abs(so.bs1770_integrated_loudness(sine, sr) - (-3.01)) < 0.05
    assert abs(so.bs1770_integrated_loudness(np.stack([sine, sine], 1), sr) - 0.0) < 0.05


@pytest.mark.parametrize("N,C,sr", [(160000, 2, 16000), (48000, 1, 16000), (5000, 2, 16000), (96000, 5, 48000),
                                    (6400, 1, 16000), (100001, 3, 16000)])
def test_emulated_kernels_match_oracle(emu, N, C, sr):
    x = stems(N + C, N, C, sr)
    block = 0.4 if N / sr >= 0.4 else N / sr
    ref = so.bs1770_integrated_loudness(x, sr, block)
    got, gain = emu.lufs(x, sr, block, target=-23.0)
    assert abs(got - ref) < 1e-4, (got, ref)                    # 1e-4 dB -> 1.2e-5 relative gain error
    assert abs(gain - 10 ** ((-23.0 - ref) / 20)) / gain < 2e-5


def test_silence_maps_to_minus_40(emu):
    x = np.zeros((16000, 2), np.float32)
    lufs, gain = emu.lufs(x, 16000, 0.4, target=-17.0)
    assert np.isinf(lufs) and lufs < 0
    assert abs(gain - 10 ** ((-17.0 + 40.0) / 20)) < 1e-9       # SonicSim_audio.py:73-75
    with np.errstate(all="ignore"):
        y, g = so.lufs_norm(x, 16000, -17.0)
    assert g == 0.0 and not y.any()


def test_gating_plan_matches_pyloudnorm_expressions():
    from sonicsim_b200.SonicSim_audio import gating_plan
    for N, sr, bs in [(960000, 16000, 0.4), (100001, 16000, 0.4), (2880000, 48000, 0.4), (5000, 16000, 5000 / 16000)]:
        lo, hi = so.bs1770_block_bounds(N, sr, bs)
        brk, blo, bhi = gating_plan(N, float(sr), float(bs))
        assert np.array_equal(brk[blo], np.minimum(lo, N)) and np.array_equal(brk[bhi], np.minimum(hi, N))
        assert np.all(np.diff(brk) > 0)


def _emu_vs_reference(emu, x, sr):
    N = x.shape[0]
    block = block_size_of(N, sr)
    assert_clear_of_gates(x, sr, block)
    ref = so.bs1770_integrated_loudness(x, sr, block, up_to_8_channels=True)
    got, gain = emu.lufs(x, sr, block, target=-23.0)
    assert abs(got - ref) <= EXACT_DB, (got, ref)
    used = -40.0 if np.isinf(got) else got
    assert abs(gain / 10 ** ((-23.0 - used) / 20) - 1) < 1e-12
    return got


def test_oracle_extension_to_eight_channels():
    """Channels 5-7 weigh 1 (the documented extension); by default more than five channels still raise like pyloudnorm,
    and five or fewer give the same value either way."""
    x = stems(3, 16000, 8)
    with pytest.raises(ValueError):
        so.bs1770_integrated_loudness(x[:, :6], 16000)
    with pytest.raises(ValueError):
        so.bs1770_integrated_loudness(np.zeros((16000, 9), np.float32), 16000, up_to_8_channels=True)
    assert so.bs1770_integrated_loudness(x[:, :5], 16000) == so.bs1770_integrated_loudness(x[:, :5], 16000, up_to_8_channels=True)
    # channel 7 alone weighs like channel 0 alone, channel 3 like 1.41 x channel 0
    def one(c):
        y = np.zeros_like(x)
        y[:, c] = x[:, 0]
        return y
    l0 = so.bs1770_integrated_loudness(one(0), 16000, up_to_8_channels=True)
    assert abs(so.bs1770_integrated_loudness(one(7), 16000, up_to_8_channels=True) - l0) < 1e-12
    assert abs(so.bs1770_integrated_loudness(one(3), 16000, up_to_8_channels=True) - (l0 + 10 * np.log10(1.41))) < 1e-9
    y, _ = so.lufs_norm(x, 16000, -20.0, up_to_8_channels=True)
    assert abs(so.bs1770_integrated_loudness(y, 16000, up_to_8_channels=True) - (-20.0)) < 1e-4


@pytest.mark.parametrize("C", range(1, 9))
def test_emulated_kernels_every_channel_count(emu, C):
    _emu_vs_reference(emu, stems(40 + C, 27001, C), 16000)


@pytest.mark.parametrize("sr", RATES)
def test_emulated_kernels_every_rate(emu, sr):
    for C in (1, 6):
        _emu_vs_reference(emu, stems(sr + C, int(2.37 * sr), C, sr), sr)


@pytest.mark.parametrize("n_e", [1, 31, 32, 33, 600])
def test_emulated_kernels_interval_counts(emu, n_e):
    """n_e = elementary intervals of a channel: one (a clip shorter than a gating block), around the 32 lanes of the
    device scan, and many per lane."""
    sr = 16000
    N = n_samples_for(n_e, sr)
    _emu_vs_reference(emu, stems(n_e, N, 2, sr), sr)


@pytest.mark.parametrize("sr", [16000, 44100])
def test_emulated_kernels_last_block_clipped_at_n(emu, sr):
    """1.06 s: round() adds a gating block whose end lies past the clip; pyloudnorm's x[l:u] clips it at N."""
    N = int(1.06 * sr)
    lo, hi = so.bs1770_block_bounds(N, sr, 0.4)
    assert hi[-1] > N and lo[-1] < N
    _emu_vs_reference(emu, stems(7, N, 3, sr), sr)


def test_emulated_kernels_do_not_depend_on_the_partition(emu, monkeypatch):
    """gating_plan(refine=k) cuts each interval into k: more, shorter per-thread recurrences, the same loudness.  The
    emulation takes its gating tables from SonicSim_audio.gating_plan, which is bound here to each refinement."""
    from sonicsim_b200 import SonicSim_audio as sa
    plan = sa.gating_plan
    for sr, N, C, signal in PARTITION_CASES:
        x = signal(N + C, N, C, sr)
        got, n_e = [], []
        for k in REFINES:
            def refined(num_samples, rate, block_size, k=k):
                brk, lo, hi = plan(num_samples, rate, block_size, k)
                n_e.append(len(brk) - 1)
                return brk, lo, hi
            monkeypatch.setattr(sa, "gating_plan", refined)
            got.append(_emu_vs_reference(emu, x, sr))
        assert n_e[-1] >= 32 * n_e[0] // 2 and n_e == sorted(n_e), n_e
        assert max(got) - min(got) < 1e-8, got


@pytest.mark.gpu
@pytest.mark.parametrize("N,C", [(480000, 2), (960000, 1), (100001, 5), (5000, 2)])
def test_gpu_lufs_norm_matches_oracle(N, C):
    from sonicsim_b200 import SonicSim_audio as sa
    x = stems(7 * N + C, N, C)
    y_ref, g_ref = so.lufs_norm(x, 16000, -17.0)
    y, g = sa.lufs_norm(x, 16000, -17.0)
    assert y.dtype == np.float32 and y.shape == x.shape
    assert so.rel_rms(y, y_ref) < 1e-4
    assert abs(g - g_ref) / abs(g_ref) < 1e-3
    np.random.seed(3)
    y2, _ = sa.get_lufs_norm_audio(x, 16000, -24)
    np.random.seed(3)
    y2_ref, _ = so.get_lufs_norm_audio(x, 16000, -24)
    assert so.rel_rms(y2, y2_ref) < 1e-4


@pytest.mark.gpu
def test_gpu_lufs_errors_like_pyloudnorm():
    from sonicsim_b200 import SonicSim_audio as sa
    with pytest.raises(ValueError):
        sa.lufs_norm(np.zeros((16000, 6), np.float32), 16000, -17)      # > 5 channels (SURVEY D5)
    with pytest.raises(ValueError):
        sa.lufs_norm(np.zeros((16000, 2), np.int16), 16000, -17)


@pytest.mark.gpu
def test_gpu_fft_conv_golden(golden):
    import torch
    from sonicsim_b200 import SonicSim_audio as sa
    g = golden("fft_conv")
    for k in range(int(g["n_cases"])):
        y = sa.fft_conv(torch.from_numpy(g[f"x{k}"]), torch.from_numpy(g[f"h{k}"]), is_cpu=True)
        assert isinstance(y, torch.Tensor) and y.shape == torch.Size(g[f"y{k}"].shape)
        assert so.rel_rms(y.numpy(), g[f"y{k}"]) < 1e-4


@pytest.mark.gpu
def test_gpu_render_scene_with_loudness_matches_reference_pipeline():
    """SonicSet.py:77-101: render 2 moving + 2 static stems, then get_lufs_norm_audio on each."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(77)
    N, C, L, P = 64000, 2, 1500, 5
    moving = [(so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)) for _ in range(2)]
    static = [(so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, L)[0]) for _ in range(2)]
    np.random.seed(123)
    ym, ys = render.render_scene(moving, static, sr=16000, moving_lufs=-17, static_lufs=[-24, -29])
    # the reference's order of RNG draws: trajectories first (interpolate_moving_audio), then the targets
    np.random.seed(123)
    stems_ref = []
    for x, h, pos in moving:
        idx, w = so.setup_dynamic_interp(pos, N)
        stems_ref.append(so.convolve_moving_receiver(x, h, idx, w))
    for x, h in static:
        stems_ref.append(so.convolve_fixed_receiver(x[None], h))
    refs = []
    for stem, l in zip(stems_ref, [-17, -17, -24, -29]):
        refs.append(so.get_lufs_norm_audio(np.ascontiguousarray(stem.T), 16000, l)[0].T)
    for y, r in zip(ym + ys, refs):
        assert so.rel_rms(y, r) < 1e-4


def test_relative_gate_known_answer(emu):
    """BS.1770 gating, analytic expectation: 10 s of a 997 Hz sine at -20 dBFS followed by 10 s at -50 dBFS.
    Both halves pass the absolute gate (-70); their mean power sets the relative gate at about -36 LKFS, which
    removes the quiet half: the integrated loudness is that of the loud half, -23.0 LKFS."""
    sr = 48000
    t = np.arange(sr * 10) / sr
    sine = np.sin(2 * np.pi * 997 * t)
    x = np.concatenate([sine * 10 ** (-20 / 20), sine * 10 ** (-50 / 20)]).astype(np.float32)
    ref = so.bs1770_integrated_loudness(x, sr)
    assert abs(ref - (-23.01)) < 0.15          # transition blocks (400 ms, partly quiet) pull it down by ~0.07 dB
    got, _ = emu.lufs(x, sr, 0.4)
    assert abs(got - ref) < 1e-4
    # without the relative gate the answer would be the mean power of both halves, ~ -26.0: the gate matters
    assert ref > -24.0


def test_oracle_loudness_close_to_torchaudio_bs1770():
    """Independent implementation of the same recommendation (torchaudio.functional.loudness, BS.1770-4): the
    oracle's restatement of pyloudnorm agrees with it within 0.3 LU on programme material with silent gaps and
    level steps, where the two gates matter (without gating the same signals read > 1 LU lower).  This is a sanity
    bound, not the pin - pyloudnorm's filter coefficients differ slightly from torchaudio's."""
    import torch
    import torchaudio
    from scipy import signal
    rng = np.random.default_rng(1)
    for sr, C in [(16000, 1), (16000, 2), (48000, 2)]:
        segs = []
        for lvl, dur in [(0.2, 2.0), (0.0, 1.5), (0.003, 2.0), (0.1, 1.0), (0.0, 0.7), (0.3, 1.3)]:
            n = int(sr * dur)
            segs.append(rng.standard_normal((n, C)) * lvl + (lvl * 0.5) * np.sin(2 * np.pi * 300 * np.arange(n) / sr)[:, None])
        x = np.concatenate(segs).astype(np.float64)
        ours = so.bs1770_integrated_loudness(x, sr)
        theirs = torchaudio.functional.loudness(torch.from_numpy(x.T.copy()).float(), sr).item()
        assert abs(ours - theirs) < 0.3, (sr, C, ours, theirs)
        y = x.copy()
        for b, a in so.bs1770_k_weighting(sr):
            y = signal.lfilter(b, a, y, axis=0)
        ungated = -0.691 + 10.0 * np.log10(np.sum(np.mean(y ** 2, axis=0)))
        assert theirs - ungated > 1.0, (sr, C, ungated, theirs)


# ---- pins against the real pyloudnorm 0.1.1: live when the package can be imported, and through the fixture
# oracle/pin_loudness.py writes when it can.  Neither is available in the authoring image (no network): both skip there
# and a5 stays "parity unpinned"; on a box that has the package they turn the restated oracle into a pinned one.
def _golden_lufs():
    import os
    p = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lufs_norm.npz")
    return np.load(p) if os.path.isfile(p) else None


def test_oracle_matches_live_pyloudnorm():
    pyln = pytest.importorskip("pyloudnorm")
    for seed, N, C, sr in [(11, 160000, 2, 16000), (12, 96000, 5, 48000), (13, 5000, 1, 16000)]:
        x = stems(seed, N, C, sr)
        block = 0.4 if N > 0.4 * sr else N / sr
        ref = pyln.Meter(rate=sr, block_size=block).integrated_loudness(x)
        assert abs(so.bs1770_integrated_loudness(x, sr, block) - ref) < 1e-9
        y_ref = pyln.normalize.loudness(x, ref, -17.0)
        assert so.rel_rms(so.lufs_norm(x, sr, -17.0)[0], y_ref) < 1e-7


def test_oracle_matches_pyloudnorm_fixture():
    g = _golden_lufs()
    if g is None:
        pytest.skip("tests/golden/lufs_norm.npz not present (oracle/pin_loudness.py could not import pyloudnorm)")
    for k in range(int(g["n_cases"])):
        N, C, sr = int(g[f"N{k}"]), int(g[f"C{k}"]), int(g[f"sr{k}"])
        x = stems(int(g[f"seed{k}"]), N, C, sr)
        y, _ = so.lufs_norm(x, sr, -17.0)
        assert so.rel_rms(y[:: max(1, N // 4096)], g[f"y{k}"]) < 1e-6


@pytest.mark.gpu
def test_gpu_lufs_norm_matches_pyloudnorm_fixture():
    g = _golden_lufs()
    if g is None:
        pytest.skip("tests/golden/lufs_norm.npz not present (oracle/pin_loudness.py could not import pyloudnorm)")
    from sonicsim_b200 import SonicSim_audio as sa
    for k in range(int(g["n_cases"])):
        N, C, sr = int(g[f"N{k}"]), int(g[f"C{k}"]), int(g[f"sr{k}"])
        x = stems(int(g[f"seed{k}"]), N, C, sr)
        y, _ = sa.lufs_norm(x, sr, -17.0)
        assert so.rel_rms(y[:: max(1, N // 4096)], g[f"y{k}"]) < 1.2e-5          # 1e-4 dB


@pytest.mark.gpu
def test_gpu_kweighting_state_is_exact_for_long_stems():
    """The three-pass K-weighting carries the exact filter state into every gating interval: a stem whose loud part is
    preceded by a strong sub-sonic transient (which a truncated warm-up would forget) still matches the oracle's
    sequential lfilter to 1e-6 dB."""
    from sonicsim_b200 import SonicSim_audio as sa
    sr, N = 16000, 16000 * 20
    rng = np.random.default_rng(5)
    x = (rng.standard_normal((N, 2)) * 0.01).astype(np.float32)
    x[: sr // 2] += 0.9                                           # DC step: excites the 38 Hz high-pass for seconds
    ref = so.bs1770_integrated_loudness(x, sr, 0.4)
    got = sa.integrated_loudness_and_norm(x, sr, 0.4, -20.0)[0]
    assert abs(got - ref) < 1e-6, (got, ref)


# ---- EBU Tech 3341 "minimum requirements" signals for the integrated loudness (the cases pyloudnorm's own test
# suite checks with the EBU wav files): synthesised here, expected values from the specification, +-0.1 LU.
def _ebu_case(case, sr=48000):
    def tone(dbfs, seconds, f=1000.0):
        t = np.arange(int(seconds * sr)) / sr
        s = (10.0 ** (dbfs / 20.0)) * np.sin(2 * np.pi * f * t)
        return np.stack([s, s], 1)
    if case == 1:
        return tone(-23.0, 20), -23.0
    if case == 2:
        return tone(-33.0, 20), -33.0
    if case == 3:                                   # relative gate: the quiet parts must be ignored
        return np.concatenate([tone(-36.0, 10), tone(-23.0, 60), tone(-36.0, 10)]), -23.0
    if case == 4:                                   # absolute gate as well
        return np.concatenate([tone(-72.0, 10), tone(-36.0, 10), tone(-23.0, 60), tone(-36.0, 10), tone(-72.0, 10)]), -23.0
    if case == 5:
        return np.concatenate([tone(-26.0, 20), tone(-20.0, 20.1), tone(-26.0, 20)]), -23.0
    raise ValueError(case)


@pytest.mark.parametrize("case", [1, 2, 3, 4, 5])
def test_oracle_and_emulated_kernels_on_ebu_3341_signals(emu, case):
    x, want = _ebu_case(case)
    x = x.astype(np.float32)
    got = so.bs1770_integrated_loudness(x, 48000, 0.4)
    assert abs(got - want) < 0.1, (case, got)
    got_emu, _ = emu.lufs(x, 48000, 0.4, target=-23.0)
    assert abs(got_emu - got) < 1e-4


@pytest.mark.gpu
@pytest.mark.parametrize("case", [1, 3, 4, 5])
def test_gpu_loudness_on_ebu_3341_signals(case):
    from sonicsim_b200 import SonicSim_audio as sa
    x, want = _ebu_case(case)
    x = x.astype(np.float32)
    got = sa.integrated_loudness_and_norm(x, 48000, 0.4, -23.0, want_output=False)[0]
    assert abs(got - want) < 0.1 and abs(got - so.bs1770_integrated_loudness(x, 48000, 0.4)) < 1e-4
