"""The loudness kernels (k_kweight<1..3>, k_kw_scan, k_loud_gate, k_loud_scale) against the float64 BS.1770
restatement of oracle/sonicsim_oracle.py, everywhere the library uses them: ss_loudness_dev called directly on
heterogeneous batches (1-8 channels, clips shorter than a gating block, both layouts, unaligned and odd-sized buffers,
every output mode) at five sample rates, the gating edges, ss_render_host_ex split into many chunks, and the argument
checks.  Loudness must match to 1e-6 dB, and every output must be exactly float32(gain) * input."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from gpu_plumbing import small_host_budget_context
from loudness_cases import (EXACT_DB, MALFORMED, PARTITION_CASES, RATES, REFINES, Stem, _reference, _scene, _stem_shape,
                            assert_clear_of_gates, block_size_of, n_samples_for, stems)

pytestmark = pytest.mark.gpu

NAN = float("nan")


def loudness_dev(stems_):
    """One ss_loudness_dev call over every stem; returns its status."""
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    arr = (_lib.SsLoudItem * len(stems_))(*[s.item for s in stems_])
    st = R.lib.ss_loudness_dev(R.ctx, arr, len(stems_), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return st


def check_stem(s, ref=None):
    """|LUFS - reference| <= 1e-6 dB, gain as pyln.normalize.loudness computes it, output == float32(gain) * x."""
    lufs, gain = s.lufs_gain()
    ref = _reference(s.x, s.sr) if ref is None else ref
    if np.isinf(ref):
        assert lufs == ref
    else:
        assert abs(lufs - ref) <= EXACT_DB, (lufs, ref, s.C, s.N, s.sr)
    used = -40.0 if np.isinf(lufs) else lufs
    assert gain == pytest.approx(10 ** ((s.target - used) / 20), rel=1e-13)
    out = s.output()
    if out is not None:
        want = np.float32(gain) * s.x                                    # float32 * float32 array: float32
        assert want.dtype == np.float32 and np.array_equal(out, want)
    return lufs, gain, out


def _batch(sr, seed):
    """Heterogeneous stems at one rate: C = 1..8, clips from 0.21 s (shorter than a gating block) to ~60 s (about
    600 intervals), N * C both a multiple of 4 and not, interleaved and channel-major, every output mode, aligned
    and unaligned buffers."""
    specs = [  # (seconds or n_e, C, layout, out, off)
        (0.21, 1, "cn", "sep", 0), (1.06, 2, "nc", "alias", 0), (("n_e", 33), 3, "cn", "sep", 1),
        (0.37, 4, "nc", "none", 1), (2.05, 5, "cn", "alias", 1), (("n_e", 31), 6, "nc", "sep", 0),
        (0.9, 7, "cn", "sep", 0), (1.6, 8, "nc", "sep", 1), (60.3, 3, "cn", "sep", 0),
    ]
    out = []
    for k, (d, C, layout, mode, off) in enumerate(specs):
        N = n_samples_for(d[1], sr) if isinstance(d, tuple) else int(d * sr) + (k % 3)
        x = stems(seed + k, N, C, sr)
        assert_clear_of_gates(x, sr, block_size_of(N, sr))
        out.append(Stem(x, sr, -30.0 + 2 * k, layout, mode, off))
    assert any(s.n % 4 for s in out) and any(s.n % 4 == 0 for s in out)
    return out


@pytest.mark.parametrize("sr", RATES)
def test_loudness_dev_heterogeneous_batch(sr):
    batch = _batch(sr, sr)
    refs = [_reference(s.x, sr) for s in batch]
    assert loudness_dev(batch) == 0
    got = [check_stem(s, r) for s, r in zip(batch, refs)]
    worst = max(abs(g[0] - r) for g, r in zip(got, refs))
    print("ss_loudness_dev at %d Hz: max |dLUFS| = %.3g dB" % (sr, worst))
    # each stem alone gives the same bits as inside the batch, in its own layout and in the other one
    for s, r, (lufs, gain, out) in zip(batch, refs, got):
        other = "nc" if s.layout == "cn" else "cn"
        for t in (Stem(s.x, sr, s.target, s.layout, s.mode, s.off), Stem(s.x, sr, s.target, other, "sep", s.off)):
            assert loudness_dev([t]) == 0
            lt, gt, ot = check_stem(t, r)
            assert lt == lufs and gt == gain
            assert out is None or np.array_equal(ot, out)


@pytest.mark.parametrize("case", range(len(PARTITION_CASES)))
def test_loudness_dev_does_not_depend_on_the_partition(case):
    """gating_plan(refine=k) cuts every interval into k.  A 0.41 s clip with refine = 32 gives 32 lanes of one 12.5 ms
    interval each: the state a lane starts in then still matters after the lane before it, so a wrong composition in
    k_kw_scan's warp scan shows in the loudness."""
    sr, N, C, signal = PARTITION_CASES[case]
    x = signal(N + C, N, C, sr)
    assert_clear_of_gates(x, sr, block_size_of(N, sr))
    ref = _reference(x, sr)
    for k in REFINES:
        s = Stem(x, sr, -23.0, "cn", "sep", 0, refine=k)
        assert loudness_dev([s]) == 0
        check_stem(s, ref)


def _copies(s, n):
    """n measure-only items over the data of Stem `s`, each with its own scratch and a NaN-filled result."""
    from sonicsim_b200 import _lib
    per = s.scratch.numel()
    scratch = torch.empty(n * per, dtype=torch.float64, device="cuda")
    res = torch.full((n, 2), NAN, dtype=torch.float64, device="cuda")
    arr = (_lib.SsLoudItem * n)()
    for i in range(n):
        it = _lib.SsLoudItem.from_buffer_copy(s.item)
        it.out, it.scratch, it.result = None, scratch.data_ptr() + 8 * per * i, res[i].data_ptr()
        arr[i] = it
    return arr, scratch, res


def test_loudness_dev_item_limit():
    """One gridDim.y row per item in k_kw_scan and k_loud_scale: 65536 items are refused (SS_ERR_UNSUPPORTED) before
    anything is written; 65535 measure-only items over one tiny stem are accepted and each gives the single item's
    result, which matches the float64 reference."""
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    sr, N = 16000, 1600
    x = stems(5, N, 1, sr)
    assert_clear_of_gates(x, sr, block_size_of(N, sr))
    one = Stem(x, sr, -23.0, "cn", "none")
    assert loudness_dev([one]) == 0
    check_stem(one)
    want = one.res.cpu().numpy()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    arr, scratch, res = _copies(one, 65536)
    assert R.lib.ss_loudness_dev(R.ctx, arr, 65536, stream) == _lib.SS_ERR_UNSUPPORTED
    torch.cuda.synchronize()
    assert torch.isnan(res).all()
    assert R.lib.ss_loudness_dev(R.ctx, arr, 65535, stream) == 0
    torch.cuda.synchronize()
    got = res.cpu().numpy()
    assert np.array_equal(got[:65535], np.broadcast_to(want, (65535, 2)))
    assert np.isnan(got[65535]).all()


def test_loudness_dev_mixed_rates_in_one_call_are_rejected():
    a = Stem(stems(1, 8000, 2, 16000), 16000, -20.0)
    b = Stem(stems(2, 24000, 2, 48000), 48000, -20.0)
    from sonicsim_b200 import _lib
    assert loudness_dev([a, b]) == _lib.SS_ERR_INVALID
    assert np.all(np.isnan(a.obuf.cpu().numpy())) and np.all(np.isnan(b.res.cpu().numpy()))


def test_loudness_dev_strides_measure_any_layout_but_scale_dense_ones_only():
    """A padded (N, C) layout - rows of C + 3 floats - is measured like the dense stem with out = NULL.  With an
    output the kernel would scale the first N*C floats of the buffer, which are not the stem: rejected up front."""
    from sonicsim_b200 import _lib
    sr, C, N = 16000, 3, 20011
    x = stems(9, N, C, sr)
    padded = np.full((N, C + 3), np.nan, np.float32)
    padded[:, :C] = x
    dev = torch.from_numpy(padded.reshape(-1)).cuda()
    s = Stem(x, sr, -20.0, "nc", "none")
    s.item.data, s.item.stride_n, s.item.stride_c = dev.data_ptr(), C + 3, 1
    assert loudness_dev([s]) == 0
    dense = Stem(x, sr, -20.0, "nc", "none")
    assert loudness_dev([dense]) == 0
    assert s.lufs_gain() == dense.lufs_gain()
    check_stem(dense)
    for mode in ("sep", "alias"):
        t = Stem(x, sr, -20.0, "nc", mode)
        t.item.data, t.item.stride_n, t.item.stride_c = dev.data_ptr(), C + 3, 1
        if mode == "alias":
            t.item.out = dev.data_ptr()
        assert loudness_dev([t]) == _lib.SS_ERR_INVALID
        assert np.all(np.isnan(t.res.cpu().numpy()))
    assert np.array_equal(dev.cpu().numpy(), padded.reshape(-1), equal_nan=True)
    # the host entry copies N*C floats as one block: non-dense strides are rejected even when measuring only
    from sonicsim_b200 import render
    from sonicsim_b200.SonicSim_audio import gating_plan
    R = render.default_renderer()
    brk, lo, hi = gating_plan(N, float(sr), 0.4)
    lufs, gain = ctypes.c_double(NAN), ctypes.c_double(NAN)
    host = np.ascontiguousarray(padded.reshape(-1))
    for out in (None, np.empty(N * (C + 3), np.float32)):
        st = R.lib.ss_lufs_norm_host(R.ctx, host.ctypes.data, None if out is None else out.ctypes.data, N, C, C + 3, 1,
                                     float(sr), 0.4, -20.0, brk.ctypes.data, len(brk) - 1, lo.ctypes.data,
                                     hi.ctypes.data, len(lo), ctypes.byref(lufs), ctypes.byref(gain))
        assert st == _lib.SS_ERR_INVALID and np.isnan(lufs.value)
    # the dense channel-major form through the host entry is fine
    xc = np.ascontiguousarray(x.T)
    st = R.lib.ss_lufs_norm_host(R.ctx, xc.ctypes.data, None, N, C, 1, N, float(sr), 0.4, -20.0, brk.ctypes.data,
                                 len(brk) - 1, lo.ctypes.data, hi.ctypes.data, len(lo), ctypes.byref(lufs),
                                 ctypes.byref(gain))
    assert st == 0 and (lufs.value, gain.value) == dense.lufs_gain()


# ---- gating edges: every signal asserts, on the reference side, that no block lies within 1e-3 dB of a gate
def _gating_signals(sr):
    rng = np.random.default_rng(sr)
    N = int(3.3 * sr)
    t = np.arange(N) / sr
    quiet = (rng.standard_normal((N, 2)) * 1e-5).astype(np.float32)              # ~ -97 LUFS: no block passes -70
    some_silent = stems(5, N, 5, sr)
    some_silent[:, [1, 3]] = 0
    sine = np.sin(2 * np.pi * 997 * t)
    steps = np.where(t < 1.5, 10 ** (-20 / 20), 10 ** (-50 / 20)) * sine       # the relative gate drops the quiet half
    steps = np.stack([steps, 0.5 * steps, steps], 1).astype(np.float32)
    return {"silent": np.zeros((N, 3), np.float32), "quiet": quiet, "some_channels_silent": some_silent,
            "relative_gate": steps}


@pytest.mark.parametrize("sr", [16000, 48000])
@pytest.mark.parametrize("name", ["silent", "quiet", "some_channels_silent", "relative_gate"])
def test_loudness_dev_gating_edges(sr, name):
    x = _gating_signals(sr)[name]
    block = block_size_of(x.shape[0], sr)
    l, gamma_r = assert_clear_of_gates(x, sr, block)
    ref = _reference(x, sr)
    if name in ("silent", "quiet"):
        assert np.isinf(ref) and ref < 0 and np.all(l < -70)
    if name == "relative_gate":
        assert np.sum(l > -70) > np.sum(l > gamma_r) > 0                     # the relative gate decides
    s = Stem(x, sr, -23.0, "nc", "sep", 1)
    assert loudness_dev([s]) == 0
    lufs, gain, out = check_stem(s, ref)
    if name == "quiet":                                                      # -inf -> -40: scaled up, not zeroed
        assert gain == pytest.approx(10 ** ((-23.0 + 40.0) / 20), rel=1e-13)
        assert np.count_nonzero(out) == np.count_nonzero(x)
    if name == "some_channels_silent":
        assert not out[:, [1, 3]].any()


# ---- ss_render_host_ex split into many chunks


def _check_scene(srcs, targets, direct, run):
    """run(lufs_targets) -> (outs, direct_out, [(lufs, gain)] or None), the same sources every time."""
    raw, raw_d, _ = run(None)
    outs, out_d, loud = run(targets)
    worst = 0.0
    for i, (s, t) in enumerate(zip(srcs, targets)):
        if t is None:
            assert np.array_equal(outs[i], raw[i]) and all(np.isnan(loud[i]))
            continue
        lufs, gain = loud[i]
        stem = np.ascontiguousarray(raw[i].T)
        assert_clear_of_gates(stem, 16000, block_size_of(stem.shape[0], 16000))
        ref = _reference(stem, 16000)
        assert abs(lufs - ref) <= EXACT_DB, (i, lufs, ref)
        worst = max(worst, abs(lufs - ref))
        assert gain == pytest.approx(10 ** ((t - lufs) / 20), rel=1e-13)
        assert np.array_equal(outs[i], np.float32(gain) * raw[i])
        if i == direct:
            assert np.array_equal(out_d, np.float32(gain) * raw_d)          # the reverberant stem's gain
    return worst


def test_render_host_ex_many_chunks_normalises_every_stem():
    """A dedicated context whose host pipeline budget is 1 MB (SS_HOST_CHUNK_MB, read by ss_create): the batch falls
    into many more chunks than there are slots and side streams, each with its own loudness call and gating tables."""
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    srcs, targets, direct = _scene(np.random.default_rng(1770))
    with small_host_budget_context() as ctx:
        def run(lufs_targets):
            outs = [np.full(_stem_shape(s), NAN, np.float32) for s in srcs]
            dd = [np.full(_stem_shape(s), NAN, np.float32) if i == direct else None for i, s in enumerate(srcs)]
            plan = R.plan_host(srcs, outs, lufs_targets, 16000, dd)          # bound here, rendered in `ctx`
            if plan.post is None:
                _lib.check(R.lib.ss_render_host(ctx, plan.items, plan.n))
            else:
                _lib.check(R.lib.ss_render_host_ex(ctx, plan.items, plan.n, plan.post))
            return outs, dd[direct], plan.loudness()
        worst = _check_scene(srcs, targets, direct, run)
    print("render_host_ex, many chunks: max |dLUFS| = %.3g dB" % worst)


def test_plan_host_heterogeneous_batch_default_context():
    from sonicsim_b200 import render
    R = render.default_renderer()
    srcs, targets, direct = _scene(np.random.default_rng(85), 9)

    def run(lufs_targets):
        dd = [np.full(_stem_shape(s), NAN, np.float32) if i == direct else None for i, s in enumerate(srcs)]
        plan = R.plan_host(srcs, None, lufs_targets, 16000, dd)
        return plan.run(), dd[direct], plan.loudness()
    worst = _check_scene(srcs, targets, direct, run)
    print("plan_host, default context: max |dLUFS| = %.3g dB" % worst)


# ---- argument checks
def _c_abi_items(rng, rates, C=2, N=24000):
    """Static sources with NaN-filled outputs and their post items; rates[i] None = no target."""
    from sonicsim_b200 import _lib
    from sonicsim_b200.SonicSim_audio import gating_plan
    keep, outs = [], []
    items = (_lib.SsSource * len(rates))()
    post = (_lib.SsPostLufs * len(rates))()
    for i, r in enumerate(rates):
        x, h = so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, 300)[0]
        out = np.full((C, N), NAN, np.float32)
        items[i] = _lib.SsSource(x=x.ctypes.data, rir=h.ctypes.data, out=out.ctypes.data, N=N, P=1, C=C, L=300,
                                 mode=_lib.SS_STATIC)
        res = np.full(2, NAN)
        if r is not None:
            brk, lo, hi = gating_plan(N, float(r), 0.4)
            post[i] = _lib.SsPostLufs(brk=brk.ctypes.data, blk_lo=lo.ctypes.data, blk_hi=hi.ctypes.data,
                                      n_e=len(brk) - 1, n_blocks=len(lo), rate=float(r), block_size=0.4,
                                      target_lufs=-20.0, result=res.ctypes.data)
            keep.append((brk, lo, hi))
        keep.append((x, h, res))
        outs.append(out)
    return items, post, outs, keep


def test_render_host_ex_rejects_mixed_rates_and_wide_stems_before_any_copy():
    """Source 0 has no target, sources 1 and 2 have targets at 16 and 48 kHz: invalid whether the three share a chunk
    (default budget) or not (a 1 MB host budget), and nothing is written.  So is a target on a 9-channel stem."""
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    rng = np.random.default_rng(4)
    with small_host_budget_context() as small:
        for ctx in (R.ctx, small):
            for rates in ([None, 16000, 48000], [16000, None, 48000], [None, 48000, None, 16000]):
                items, post, outs, keep = _c_abi_items(rng, rates, N=96000)
                assert R.lib.ss_render_host_ex(ctx, items, len(rates), post) == _lib.SS_ERR_INVALID
                assert all(np.all(np.isnan(o)) for o in outs)
            items, post, outs, keep = _c_abi_items(rng, [None, 16000, 16000], N=96000)
            assert R.lib.ss_render_host_ex(ctx, items, 3, post) == 0
            items, post, outs, keep = _c_abi_items(rng, [16000], C=9)
            assert R.lib.ss_render_host_ex(ctx, items, 1, post) == _lib.SS_ERR_INVALID
            assert np.all(np.isnan(outs[0]))
            items, post, outs, keep = _c_abi_items(rng, [None], C=9)                 # no target: 9 channels render
            assert R.lib.ss_render_host_ex(ctx, items, 1, post) == 0
    # the Python layer
    x, h = so.synth_dry(rng, 16000), so.synth_rirs(rng, 1, 9, 300)[0]
    with pytest.raises(ValueError):
        R.render_host([render.StaticSource(x, h)], lufs_targets=[-20.0])
    from sonicsim_b200 import SonicSim_audio as sa
    with pytest.raises(ValueError):
        sa.integrated_loudness_and_norm(np.zeros((16000, 9), np.float32), 16000, 0.4, -20.0)


# one malformed field of an ss_post_lufs entry with a target (ctypes: None is a NULL pointer)


def _results(post, i):
    return np.frombuffer((ctypes.c_double * 2).from_address(post[i].result), np.float64)


@pytest.mark.parametrize("bad", list(MALFORMED))
def test_render_host_ex_rejects_each_malformed_entry_before_any_copy(bad):
    """The third of three sources (the first has no target) has one malformed field: ss_render_host_ex refuses the call
    whether the sources share a chunk or not, and writes no output and no result.  ss_lufs_norm_host refuses the same
    gating arguments."""
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    rng = np.random.default_rng(5)
    field, value = MALFORMED[bad]
    with small_host_budget_context() as small:
        for ctx in (R.ctx, small):
            items, post, outs, keep = _c_abi_items(rng, [None, 16000, 16000], N=96000)
            setattr(post[2], field, value)
            assert R.lib.ss_render_host_ex(ctx, items, 3, post) == _lib.SS_ERR_INVALID
            assert all(np.all(np.isnan(o)) for o in outs)
            assert all(np.all(np.isnan(_results(post, i))) for i in (1, 2))
    q = post[2]
    N, C = 96000, 2
    x = so.synth_dry(rng, N * C)
    out = np.full(N * C, NAN, np.float32)
    lufs, gain = ctypes.c_double(NAN), ctypes.c_double(NAN)
    st = R.lib.ss_lufs_norm_host(R.ctx, x.ctypes.data, out.ctypes.data, N, C, C, 1, q.rate, q.block_size, -20.0, q.brk,
                                 q.n_e, q.blk_lo, q.blk_hi, q.n_blocks, ctypes.byref(lufs), ctypes.byref(gain))
    assert st == _lib.SS_ERR_INVALID
    assert np.isnan(lufs.value) and np.isnan(gain.value) and np.all(np.isnan(out))


@pytest.mark.parametrize("targets, sr, match", [
    ([-20.0], 16000, "entries in lufs_targets"),
    ([-20.0, None, -20.0, -20.0], 16000, "entries in lufs_targets"),
    ([-20.0, NAN, None], 16000, "not finite"),
    ([float("inf"), -20.0, None], 16000, "not finite"),
    ([-20.0, None, -20.0], 0, "sr must be > 0"),
    ([-20.0, None, -20.0], NAN, "sr must be > 0"),
])
def test_plan_host_refuses_bad_targets_before_any_call(targets, sr, match):
    """The wrong number of targets, a target that is not finite and sr <= 0 raise ValueError through plan_host,
    render_host and render_scene, and nothing is rendered."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    rng = np.random.default_rng(6)
    srcs = [render.StaticSource(so.synth_dry(rng, 16000), so.synth_rirs(rng, 1, 2, 300)[0]) for _ in range(3)]
    outs = [np.full((2, 16000), NAN, np.float32) for _ in srcs]
    with pytest.raises(ValueError, match=match):
        R.plan_host(srcs, outs, targets, sr)
    with pytest.raises(ValueError, match=match):
        R.render_host(srcs, outs, targets, sr)
    assert all(np.all(np.isnan(o)) for o in outs)
    if match == "sr must be > 0":                            # render_scene draws its targets itself, one per stem
        with pytest.raises(ValueError, match=match):
            render.render_scene([], [(s.dry, s.rir) for s in srcs], sr=sr, static_lufs=[-20.0] * 3)
