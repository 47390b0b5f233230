"""The mixture and overlap kernels (ss_mix_dev: k_mix_energy, k_mix_gain, k_mix_speech_energy, k_mix_write;
ss_overlap_dev: k_overlap) called through the C ABI, against tests/mix_reference.py: every float32 gain within 3 ulps
of the float64 gain, and every output bit for bit the float32 composition with those gains.  Every buffer sits inside
a NaN-filled allocation, at 0-3 floats past a guard, and the guards must stay NaN."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from mix_reference import F32, assert_clear_of_f32_midpoint, mix_gains_f64, overlap_exact
from gpu_plumbing import _stream, renderer
from mix_reference import MAX_ULPS, Mix, MixBuf, check_mix, mix_dev

pytestmark = pytest.mark.gpu

NAN = float("nan")
SS_ERR_INVALID, SS_ERR_UNSUPPORTED = -1, -5


def run_and_check(cases):
    """One ss_mix_dev call; every item checked.  A "null" item is checked against a "sep" twin in the same call."""
    twins = [Mix(c.spk, c.noise, c.sirs, c.snr, c.delay, "sep") if c.mode == "null" else None for c in cases]
    assert mix_dev(cases + [t for t in twins if t]) == 0
    res = []
    for c, t in zip(cases, twins):
        mix, out = c.outputs()
        if t is not None:
            tmix, tout = t.outputs()
            assert np.array_equal(mix, tmix)
            mix, out = tmix, tout
        res.append((mix, out, check_mix(c, mix, out)))
    return res


def stems(rng, S, E, scale=0.1):
    return (rng.standard_normal((S, E)) * scale * rng.uniform(0.2, 2.0, (S, 1))).astype(F32)


E_CASES = [1, 2, 3, 4, 5, 7, 4095, 4096, 4097, 65535, 65537]


@pytest.mark.parametrize("E", E_CASES)
def test_mix_items_match_composition(E):
    """S in {1, 2, 3, 8} x M in {1, 2, 8} in one call: every output mode, 0-3 float offsets, overlap shifts
    {0, 1, E - 1, E, E + 5} with M > 1, SNR in {-10, 0, 15, 20}."""
    rng = np.random.default_rng(E)
    cases = []
    for i, (S, M) in enumerate(itertools.product((1, 2, 3, 8), (1, 2, 8))):
        delay = (0, 1, E - 1, E, E + 5)[i % 5] if M > 1 else 0
        cases.append(Mix(stems(rng, S, E), stems(rng, M, E, 0.05), rng.uniform(-6, 6, max(S - 1, 1)),
                         (-10, 0, 15, 20)[i % 4], max(delay, 0), ("sep", "alias", "null")[i % 3],
                         tuple(int(v) for v in rng.integers(0, 4, 4))))
    for mode in ("sep", "alias"):                                                          # aligned: float4 path
        cases.append(Mix(stems(rng, 3, E), stems(rng, 2, E), [2.5, -4.0], 15.0, 0, mode))
    run_and_check(cases)


def test_mix_configs2_scale():
    """One item at configs[2] scale (C = 6, N = 960000), on the float4 path and on the scalar path."""
    rng = np.random.default_rng(2)
    E = 6 * 960000
    spk, noise = stems(rng, 2, E), stems(rng, 2, E, 0.03)
    run_and_check([Mix(spk, noise, [3.5], 12.0, 0, "sep")])
    run_and_check([Mix(spk, noise, [3.5], 12.0, 0, "alias", (1, 2, 3, 0))])


def test_mix_gain_edges():
    rng = np.random.default_rng(7)
    E = 4096
    a, b = stems(rng, 1, E)[0], stems(rng, 1, E)[0]
    n = stems(rng, 2, E, 0.05)
    z = np.zeros(E, F32)
    # an interferer 100 dB quieter: its gain clamps at +40 dB, exactly 100.0f
    [(mix, out, (g, gn))] = run_and_check([Mix(np.stack([a, b * F32(1e-5)]), n, [0.0], 15.0)])
    assert g[1] == F32(100.0) and np.array_equal(out[1], (b * F32(1e-5)) * F32(100.0))
    # noise 100 dB under the speech at SNR 0: the noise gain clamps at 100.0f
    [(mix, out, (g, gn))] = run_and_check([Mix(np.stack([a]), n * F32(1e-5), [], 0.0)])
    assert gn == F32(100.0)
    # the 1e-20 floor: a silent reference, a silent interferer, silent noise, all silent
    cases = [Mix(np.stack([z, b]), n, [1.0], 10.0), Mix(np.stack([a, z]), n, [1.0], 10.0),
             Mix(np.stack([a, b]), np.stack([z, z]), [1.0], 10.0, 3), Mix(np.stack([z, z, z]), np.stack([z]), [1, 2], 5.0)]
    res = run_and_check(cases)
    for mix, out, _ in res:
        assert np.all(np.isfinite(mix)) and np.all(np.isfinite(out))
    assert not res[3][0].any() and not res[3][1].any()


def test_mix_float4_and_scalar_paths_identical():
    """The same data at an aligned base (float4 path) and at a one-float offset (scalar path): identical bits.
    The midpoint guard keeps the float64 reference gains clear of float32 rounding ties; it does not bound the
    device's own double gains, which differ from the reference by up to about 1e-7 relative (the kernels square in
    float before widening).  The two paths' double gains differ only in the order of their double sums (about 1e-16
    relative), so at these fixed seeds a tie between them would fail every run, not flake."""
    rng = np.random.default_rng(11)
    for S, M, E in ((2, 1, 4096), (3, 2, 65536), (8, 8, 1024), (1, 3, 40000)):
        spk, noise, sirs, snr = stems(rng, S, E), stems(rng, M, E, 0.05), rng.uniform(-6, 6, max(S - 1, 1)), 10.0
        g64, gn64 = mix_gains_f64(spk, noise, sirs, snr)
        for v in list(g64[1:]) + [gn64]:
            assert_clear_of_f32_midpoint(v)
        aligned, shifted = run_and_check([Mix(spk, noise, sirs, snr, 0, "sep"),
                                          Mix(spk, noise, sirs, snr, 0, "sep", (1, 1, 1, 1))])
        assert np.array_equal(aligned[0], shifted[0]) and np.array_equal(aligned[1], shifted[1])


def _batch(rng):
    specs = []
    for i in range(24):
        S, M = (1, 2, 3, 5, 8)[i % 5], (1, 2, 4, 8)[i % 4]
        E = int(rng.choice([4096, 4097, 1000, 12000, 3]))
        off = (0, 0, 0, 0) if i % 2 == 0 else tuple(int(v) for v in rng.integers(0, 4, 4))
        delay = int(rng.choice([0, 1, 7, E - 1])) if M > 1 else 0
        specs.append((stems(rng, S, E), stems(rng, M, E, 0.05), rng.uniform(-6, 6, max(S - 1, 1)),
                      float(rng.uniform(-10, 20)), delay, ("sep", "alias")[i % 2], off))
    return specs


def test_mix_heterogeneous_batch_equals_single_calls():
    rng = np.random.default_rng(24)
    specs = _batch(rng)
    batch = run_and_check([Mix(*s) for s in specs])
    again = [Mix(*s) for s in specs]
    assert mix_dev(again) == 0
    for s, (mix, out, _), c in zip(specs, batch, again):
        m2, o2 = c.outputs()
        assert np.array_equal(mix, m2) and np.array_equal(out, o2)
        [(m1, o1, _)] = run_and_check([Mix(*s)])
        assert np.array_equal(mix, m1) and np.array_equal(out, o1)


def test_mix_host_entry_points_equal_dev():
    from sonicsim_b200 import mix as smix
    rng = np.random.default_rng(5)
    spk, noise = stems(rng, 3, 2 * 5001).reshape(3, 2, 5001), stems(rng, 2, 2 * 5001, 0.05).reshape(2, 2, 5001)
    m, s = smix.mix_stems(torch.from_numpy(spk), torch.from_numpy(noise), [1.5, -2.0], 14.0)
    [(dm, ds, _)] = run_and_check([Mix(spk.reshape(3, -1), noise.reshape(2, -1), [1.5, -2.0], 14.0, 0, "alias")])
    assert np.array_equal(m.numpy().reshape(-1), dm) and np.array_equal(s.numpy().reshape(3, -1), ds)
    sp, nz = stems(rng, 1, 16000)[0], stems(rng, 3, 16000, 0.05)
    m = smix.mix_noisy(torch.from_numpy(sp), torch.from_numpy(nz), -3.0, sample_rate=1000, delay=6)
    [(dm, _, _)] = run_and_check([Mix(sp[None], nz, [], -3.0, 6000, "null")])
    assert np.array_equal(m.numpy(), dm)


def _utterance(seed):
    from oracle import sonicsim_oracle as so
    rng = np.random.default_rng(seed)
    N, C, L, P = 24000, 2, 800, 4
    return {"speakers": [(so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)) for _ in range(3)],
            "noises": [(so.synth_dry(rng, N) * 0.3, so.synth_rirs(rng, 1, C, L)[0]) for _ in range(2)],
            "sirs": np.array([2.0, -3.5], np.float32), "snr": 12.0}


def test_render_mixtures_is_the_composition_of_its_stems():
    """render_mixtures' mixture is compose_mix of the stems render_device makes from the same sources, with the
    recovered gains, bit for bit.  The trajectories' sample counts are drawn from the global NumPy RNG, as the
    reference draws them, so both sides seed it identically; a second call with the same seed gives the same bits."""
    from sonicsim_b200 import render
    us = [_utterance(31), _utterance(32)]
    np.random.seed(7)
    got = render.render_mixtures(us)
    np.random.seed(7)
    again = render.render_mixtures(us)
    np.random.seed(7)
    srcs, shapes = [], []
    for u in us:
        for d, h, pos in u["speakers"]:
            b = render.trajectory_bounds(pos, d.shape[0])
            srcs.append(render.MovingSource(torch.from_numpy(d).cuda(), torch.from_numpy(h).cuda(),
                                            torch.from_numpy(b).cuda(), b))
        for d, h in u["noises"]:
            srcs.append(render.StaticSource(torch.from_numpy(d).cuda(), torch.from_numpy(h).cuda()))
    outs = [torch.full((2, 24000), NAN, device="cuda") for _ in srcs]
    render.default_renderer().render_device(srcs, outs)
    torch.cuda.synchronize()
    st = np.stack([o.cpu().numpy().reshape(-1) for o in outs])
    for k, u in enumerate(us):
        assert np.array_equal(got[k]["mix"], again[k]["mix"])
        assert np.array_equal(got[k]["speakers"], again[k]["speakers"])
        s = st[5 * k:5 * k + 5]
        c = Mix(s[:3], s[3:], u["sirs"], u["snr"])
        check_mix(c, got[k]["mix"].reshape(-1), got[k]["speakers"].reshape(3, -1))


# ---- argument checks: refused before any copy or launch, outputs untouched
def _untouched(c):
    return all(np.all(np.isnan(b.t.cpu().numpy())) for b in c.bufs() if b is not c.b_spk and b is not c.b_noise
               and b is not c.b_sirs)


def test_mix_refuses_overlapping_ranges():
    """Every range of the item lies in one NaN arena, so every overlapping variant stays inside it."""
    from sonicsim_b200 import _lib as L
    rng = np.random.default_rng(3)
    S, M, E = 2, 2, 1000
    arena = torch.full((16 * E,), NAN, device="cuda")
    arena[2 * E:4 * E] = torch.from_numpy(stems(rng, S, E).reshape(-1)).cuda()
    arena[5 * E:7 * E] = torch.from_numpy(stems(rng, M, E).reshape(-1)).cuda()
    arena[13 * E] = 1.0
    at = lambda i: arena.data_ptr() + 4 * i                      # noqa: E731
    spk, noise, mix, out, sirs, scr = at(2 * E), at(5 * E), at(8 * E), at(10 * E), at(13 * E), at(14 * E)
    base = dict(speakers=spk, noises=noise, sirs=sirs, mix=mix, speakers_out=out, scratch=scr, E=E, S=S, M=M,
                snr=10.0, noise_delay=0)
    item = lambda **kw: L.SsMixItem(**{**base, **kw})           # noqa: E731
    bad = [item(mix=spk + 4 * (E + 3)),                         # mix inside the speakers
           item(mix=noise + 4 * (2 * E - 1)),                   # mix's first float is the noises' last
           item(mix=out + 4 * E),                               # mix inside speakers_out
           item(speakers_out=spk + 4),                          # speakers_out overlaps speakers without aliasing them
           item(speakers_out=noise),                            # speakers_out on the noises
           item(speakers_out=mix - 4 * (S * E - 1)),            # speakers_out's last float is mix's first
           item(scratch=mix),                                   # scratch on the mix
           item(speakers_out=spk, mix=spk + 4 * (2 * E - 1))]   # in place, and mix meets the speakers
    R = renderer()
    before = arena.cpu().numpy()
    for it in bad:
        arr = (L.SsMixItem * 2)(item(), it)
        assert R.lib.ss_mix_dev(R.ctx, arr, 2, _stream()) == SS_ERR_INVALID
        torch.cuda.synchronize()
        assert np.array_equal(arena.cpu().numpy(), before, equal_nan=True)
    for it in (item(speakers_out=spk), item(speakers_out=None)):   # the allowed alias, and no speakers_out
        assert R.lib.ss_mix_dev(R.ctx, (L.SsMixItem * 1)(it), 1, _stream()) == 0
        torch.cuda.synchronize()
    assert np.all(np.isfinite(arena[8 * E:9 * E].cpu().numpy()))


def test_mix_limits():
    from sonicsim_b200 import _lib as L
    rng = np.random.default_rng(4)
    c = Mix(stems(rng, 1, 64), stems(rng, 1, 64), [], 10.0, 0, "null")
    R = renderer()
    arr = (L.SsMixItem * 65536)(*([c.item] * 65536))
    assert R.lib.ss_mix_dev(R.ctx, arr, 65536, _stream()) == SS_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert _untouched(c)
    # the host entry refuses before it uploads anything: E is far beyond any allocation, so only an upfront
    # refusal can return these codes
    x = np.zeros(16, F32)
    mix = np.full(16, np.nan, F32)
    E = 1 << 40
    assert R.lib.ss_mix_host_ex(R.ctx, x.ctypes.data, x.ctypes.data, None, 10.0, mix.ctypes.data, None, 2, 1, E, 0) \
        == SS_ERR_INVALID
    assert R.lib.ss_mix_host_ex(R.ctx, x.ctypes.data, x.ctypes.data, x.ctypes.data, 10.0, mix.ctypes.data, None, 9, 1,
                                E, 0) == SS_ERR_UNSUPPORTED
    assert R.lib.ss_mix_host_ex(R.ctx, x.ctypes.data, x.ctypes.data, x.ctypes.data, 10.0, mix.ctypes.data, None, 2, 9,
                                E, 0) == SS_ERR_UNSUPPORTED
    assert np.all(np.isnan(mix))


# ---- ss_overlap_dev
def overlap_dev(x, y, rows, T, D):
    R = renderer()
    st = R.lib.ss_overlap_dev(R.ctx, ctypes.c_void_p(x), ctypes.c_void_p(y), rows, T, D, _stream())
    torch.cuda.synchronize()
    return st


@pytest.mark.parametrize("rows,T", list(itertools.product((1, 3, 257), (1, 2, 5, 4097, 96001))))
def test_overlap_matches_exact(rows, T):
    rng = np.random.default_rng(rows * 7 + T)
    x = rng.standard_normal((rows, T)).astype(F32)
    for i, D in enumerate((0, 1, T - 1, T, T + 3, 1 << 40)):
        bx, by = MixBuf(rows * T, i % 4, x), MixBuf(rows * T, (i + 1) % 4)
        assert overlap_dev(bx.ptr, by.ptr, rows, T, D) == 0
        assert bx.guards_nan() and by.guards_nan() and np.array_equal(bx.get(), x.reshape(-1))
        assert np.array_equal(by.get().reshape(rows, T), overlap_exact(x, D)), (rows, T, D)


def test_overlap_limits():
    rng = np.random.default_rng(1)
    x = rng.standard_normal(65536).astype(F32)
    bx, by = MixBuf(65536, 0, x), MixBuf(65536, 1)
    assert overlap_dev(bx.ptr, by.ptr, 65535, 1, 0) == 0
    assert np.array_equal(by.get()[:65535], x[:65535] * F32(3)) and np.isnan(by.get()[65535])
    by = MixBuf(65536)
    assert overlap_dev(bx.ptr, by.ptr, 65536, 1, 0) == SS_ERR_UNSUPPORTED
    # y overlapping x without being x: refused, y untouched (x in the middle of one buffer, every y inside it)
    b = MixBuf(900, 0, rng.standard_normal(900).astype(F32))
    before = b.t.cpu().numpy()
    x0 = b.ptr + 4 * 300
    for shift in (1, 4, 299, -1, -299):
        assert overlap_dev(x0, x0 + 4 * shift, 3, 100, 2) == SS_ERR_INVALID
    assert overlap_dev(x0, x0, 3, 100, 2) == SS_ERR_INVALID
    assert np.array_equal(b.t.cpu().numpy(), before, equal_nan=True)
    assert np.all(np.isnan(by.t.cpu().numpy()))


def test_report_largest_gain_error():
    """Runs last in this module: the largest gain error the checks above met, in float32 steps."""
    print("largest gain error: %d float32 ulps" % MAX_ULPS[0])
    assert MAX_ULPS[0] <= 3
