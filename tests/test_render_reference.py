"""The float64 render reference and the local rounding scale of tests/render_reference.py, pinned on the CPU: against a
direct time-domain sum on small shapes of every mode, against the oracle's restatement of the reference on a mid-size
case, and on inputs whose scale can be computed by hand."""
import math

import numpy as np
import pytest

import render_reference as rr
from oracle import sonicsim_oracle as so


def direct_sum(x, h, idx=None, w=None):
    """y[c, n] = sum_k hat(n, p) h[p, c, k] x[n - k], summed term by term in float64 (hats 1 - w rounded to float32,
    as the reference computes them)."""
    x = np.asarray(x, np.float64)
    h = np.asarray(h, np.float64)
    h = h[None] if h.ndim == 2 else h
    P, C, L = h.shape
    N = x.size
    y = np.zeros((C, N))
    for n in range(N):
        k = np.arange(min(L, n + 1))
        hats = {0: 1.0} if idx is None else {int(idx[n]): float(np.float32(1) - np.float32(w[n])),
                                             int(idx[n]) + 1: float(w[n])}
        for p, f in hats.items():
            y[:, n] += f * (h[p][:, k] @ x[n - k])
    return y


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("N,L", [(1, 1), (7, 3), (300, 50), (200, 260)])
def test_render_f64_matches_direct_sum(mode, N, L):
    rng = np.random.default_rng(N * 7 + L + mode)
    P, C = (1 if mode == 0 else 4), 3
    x, h = so.synth_dry(rng, N), rng.standard_normal((P, C, L)).astype(np.float32)
    bounds = idx = w = None
    if mode == 1:
        cut = np.sort(rng.integers(0, N + 1, P - 2))
        bounds = np.concatenate([[0], cut, [N]]).astype(np.int32)         # empty segments allowed
        idx, w = rr.trajectory(bounds)
    elif mode == 2:
        idx = rng.integers(0, P - 1, N)
        w = rng.random(N).astype(np.float32)
    ref = direct_sum(x, h, idx, w)
    y = rr.render_f64(x, h if mode else h[0], mode, bounds=bounds, idx=idx, w=w)
    assert np.abs(y - ref).max() <= 1e-12 * max(1.0, np.abs(ref).max())
    for a, n in ((0, N), (N // 3, max(1, N // 2)), (N - 1, 1)):           # the window trick
        if a + n <= N:
            yw = rr.render_f64(x, h if mode else h[0], mode, bounds=bounds, idx=idx, w=w, window=(a, n))
            assert np.abs(yw - ref[:, a:a + n]).max() <= 1e-12 * max(1.0, np.abs(ref).max())


def test_trajectory_is_setup_dynamic_interp():
    rng = np.random.default_rng(4)
    pos = so.synth_path(rng, 9)
    np.random.seed(3)
    idx, w = so.setup_dynamic_interp(pos, 50000)
    i2, w2 = rr.trajectory(rr.bounds_from_lengths(np.bincount(idx, minlength=8)))
    assert np.array_equal(idx, i2) and np.array_equal(w, w2)


def test_render_f64_matches_reference_restatement():
    """Mid-size moving source: the float64 segment-local form equals the reference's oaconvolve + gather + lerp (in
    float64) to float64 rounding, whole and windowed."""
    rng = np.random.default_rng(11)
    P, C, L, N = 7, 3, 5000, 60000
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
    np.random.seed(2)
    idx, w = so.setup_dynamic_interp(pos, N)
    ref = so.convolve_moving_receiver(x.astype(np.float64), h.astype(np.float64), idx, w)
    y = rr.render_f64(x, h, 2, idx=idx, w=w)
    assert so.rel_rms(y, ref) < 1e-12
    bounds = rr.bounds_from_lengths(np.bincount(idx, minlength=P - 1))
    yw = rr.render_f64(x, h, 1, bounds=bounds, window=(20000, 9000))
    assert so.rel_rms(yw, ref[:, 20000:29000]) < 1e-12


def test_error_scale_by_hand():
    """White-box values: a constant dry signal and single-tap rows give norms that can be written down."""
    N = 3 * rr.B
    x = np.full(N, 2.0)
    h = np.zeros((3, 2, 10))
    h[0, 0, 0], h[1, 0, 0], h[2, 0, 0] = 1.0, 3.0, 0.5          # channel 0: norms 1, 3, 0.5 per position
    h[:, 1, 0] = 0.25                                            # channel 1: 0.25 everywhere
    pos = np.zeros(N, np.int64)                                  # every sample between positions 0 and 1
    s = rr.error_scale(x, h, pos)
    # sample n: x over [n - 12288, n + 8192) clipped to [0, N) -> min(N, n + 8192) samples of value 2
    n = np.arange(N)
    xn = 2.0 * np.sqrt(np.minimum(N, n + 8192))
    # positions idx - 1 .. idx + 2 = {0, 1, 2}; row partners (2r, 2r + 1) pair (0,0)-(0,1), (1,0)-(1,1), (2,0)-(2,1)
    assert np.allclose(s[0], xn * 3.0 / math.sqrt(8192))
    assert np.allclose(s[1], xn * 3.0 / math.sqrt(8192))        # channel 1 carries row (1, 0)'s partner error
    # static: channel pairs share a transform; a silent dry signal has scale 0
    hs = np.zeros((3, 10))
    hs[0, 0], hs[1, 0], hs[2, 0] = 1.0, 2.0, 4.0
    ss = rr.error_scale(x, hs)
    assert np.allclose(ss[0], xn * 2.0 / math.sqrt(8192)) and np.allclose(ss[2], xn * 4.0 / math.sqrt(8192))
    assert not rr.error_scale(np.zeros(N), hs).any()
    # a second partition adds the dry norm one block earlier
    hl = np.zeros((1, 1, rr.B + 1))
    hl[0, 0, 0], hl[0, 0, rr.B] = 1.0, 1.0
    sl = rr.error_scale(x, hl)
    assert np.allclose(sl[0], (xn + 2.0 * np.sqrt(np.minimum(N, n + 4096))) / math.sqrt(8192))
    # windows give the same values
    assert np.array_equal(rr.error_scale(x, h, pos, window=(5000, 300)), s[:, 5000:5300])


def test_check_render_reports_a_local_fault():
    """One wrong sample in a long stem: invisible in the global RMS, caught and located by the local check."""
    rng = np.random.default_rng(5)
    N = 40000
    x, h = so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 3000)[0]
    y64, scale = rr.render_check_inputs(x, h, 0)
    y = y64.astype(np.float32)
    worst, g = rr.check_render(y, y64, scale, 1e-6, 1e-6)
    assert worst < 1e-6 and g < 1e-7
    y[1, 2 * rr.B + 17] += 1e-4 * scale[1, 2 * rr.B + 17]
    assert so.rel_rms(y, y64) < 1e-6
    with pytest.raises(AssertionError, match=r"channel 1, sample 8209 \(tile 2\)"):
        rr.check_render(y, y64, scale, 1e-5, 1e-6)


def test_structured_inputs():
    rng = np.random.default_rng(6)
    x = rr.graded_dry(rng, 10 * rr.B + 5)
    lv = [np.abs(x[b:b + rr.B]).max() for b in range(0, x.size, rr.B)]
    assert lv[0] > 0 and min(lv) == 0 and max(lv) / min(v for v in lv if v > 0) > 2 ** 6
    h, d = rr.delay_rirs(rng, 4, 3, 9000)
    assert set(d.reshape(-1)) == set(rr.delay_taps(9000)) == {0, 1, 4095, 4096, 4097, 8999}
    g = h.reshape(12, -1).sum(axis=1)
    assert len(set(np.abs(g))) == 12 and np.count_nonzero(h) == 12
    xi = rr.impulse_dry(5000)
    assert np.count_nonzero(xi) == 6 and xi[3] == 1.0 and xi[1000] == -0.5
