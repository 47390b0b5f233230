"""Direct-path target (SS_DIRECT_TARGET) through the real kernels: one source rendering its reverberant and its
direct-path stem in the same launches equals, bit for bit, the source without the flag plus the truncated RIRs
rendered as a second source in the same kind of call - on the host path, the device path and a device plan (CUDA
graph) - and both stems match the reference's render.  Also BASELINE configs[4] at full size, the loudness gain the
direct stem shares with its reverberant stem, and the argument checks of the C ABI and the Python layer."""
import ctypes

import numpy as np
import pytest
import torch

from conftest import TOL
from direct_path import CASES, direct_path_rirs, make_case, normalized, oracle_render
from oracle import sonicsim_oracle as so

pytestmark = pytest.mark.gpu

API_CASES = [n for n in CASES if CASES[n][0] != 2]          # the Python sources take trajectory bounds only


def _sources(x, h, bounds, normalize, taps, to=lambda a: a):
    """(dual source, the same without direct_taps, the truncated RIRs as a source of their own)."""
    from sonicsim_b200 import render
    hd = direct_path_rirs(normalized(h) if normalize else h, taps)
    if bounds is None:
        mk = lambda r, nrm, t: render.StaticSource(to(x), to(r[0]), nrm, t)
    else:
        mk = lambda r, nrm, t: render.MovingSource(to(x), to(r), to(bounds), bounds, nrm, t)
    return mk(h, normalize, taps), mk(h, normalize, 0), mk(hd, False, 0), hd


def _check(out, out_d, ref, ref_d, x, h, hd, idx, w, normalize):
    assert np.array_equal(out, ref)
    assert np.array_equal(out_d, ref_d)
    assert so.rel_rms(out, oracle_render(x, normalized(h) if normalize else h, idx, w)) < TOL
    assert so.rel_rms(out_d, oracle_render(x, hd, idx, w)) < TOL


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("name", API_CASES)
def test_host_path(name, normalize):
    from sonicsim_b200 import render
    R = render.default_renderer()
    x, h, idx, w, bounds, taps = make_case(name)
    dual, plain, sep, hd = _sources(x, h, bounds, normalize, taps)
    C, N = h.shape[1], x.shape[0]
    out_d = np.full((C, N), np.nan, np.float32)
    out = R.render_host([dual], direct_outs=[out_d])[0]
    ref, ref_d = R.render_host([plain, sep])
    _check(out, out_d, ref, ref_d, x, h, hd, idx, w, normalize)


@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("name", API_CASES)
def test_device_path_and_plan(name, normalize):
    from sonicsim_b200 import render
    R = render.default_renderer()
    x, h, idx, w, bounds, taps = make_case(name)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dual, plain, sep, hd = _sources(x, h, bounds, normalize, taps, to)
    C, N = h.shape[1], x.shape[0]
    new = lambda: torch.full((C, N), float("nan"), device="cuda")
    out, out_d, ref, ref_d = new(), new(), new(), new()
    R.render_device([dual], [out], direct_outs=[out_d])
    R.render_device([plain, sep], [ref, ref_d])
    torch.cuda.synchronize()
    host = lambda t: t.cpu().numpy()
    _check(host(out), host(out_d), host(ref), host(ref_d), x, h, hd, idx, w, normalize)
    # bound once, run twice (captured into a CUDA graph on the first run, replayed on the second)
    p_dual = R.plan_device([dual], [out], direct_outs=[out_d])
    p_ref = R.plan_device([plain, sep], [ref, ref_d])
    first = []
    for k in range(2):
        for t in (out, out_d, ref, ref_d):
            t.fill_(float("nan"))
        p_dual.run(); p_ref.run()
        torch.cuda.synchronize()
        res = [host(t) for t in (out, out_d, ref, ref_d)]
        _check(*res, x, h, hd, idx, w, normalize)
        if k == 0:
            first = res
        else:
            assert all(np.array_equal(a, b) for a, b in zip(first, res))
    assert p_dual.is_graph()
    p_dual.close(); p_ref.close()


def _indexed_item(x, h, idx, w, out, flags=0, out_direct=None, taps=0):
    from sonicsim_b200 import _lib
    P, C, L = h.shape
    return _lib.SsSource(x=x.ctypes.data, rir=h.ctypes.data, out=out.ctypes.data, idx=idx.ctypes.data, w=w.ctypes.data,
                         N=x.shape[0], P=P, C=C, L=L, mode=_lib.SS_MOVING_INDEXED, flags=flags,
                         out_direct=out_direct.ctypes.data if out_direct is not None else None, direct_taps=taps)


@pytest.mark.parametrize("normalize", [False, True])
def test_indexed_trajectory_through_the_c_abi(normalize):
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    x, h, idx, w, _, taps = make_case("indexed")
    hd = direct_path_rirs(normalized(h) if normalize else h, taps)
    C, N = h.shape[1], x.shape[0]
    out, out_d, ref, ref_d = (np.full((C, N), np.nan, np.float32) for _ in range(4))
    nrm = _lib.SS_RIR_NORMALIZE if normalize else 0
    one = (_lib.SsSource * 1)(_indexed_item(x, h, idx, w, out, nrm | _lib.SS_DIRECT_TARGET, out_d, taps))
    _lib.check(R.lib.ss_render_host(R.ctx, one, 1))
    two = (_lib.SsSource * 2)(_indexed_item(x, h, idx, w, ref, nrm), _indexed_item(x, hd, idx, w, ref_d))
    _lib.check(R.lib.ss_render_host(R.ctx, two, 2))
    _check(out, out_d, ref, ref_d, x, h, hd, idx, w, normalize)


def test_cfg5_enhancement_mixture_as_one_dual_source():
    """BASELINE configs[4]: 1 moving speaker (binaural, P = 40, 60 s) with its 2.5 ms direct-path target, noise and
    music, in one call."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(5001)
    N, C, L, P, sr = 960000, 2, 4096, 40, 16000
    taps = int(0.0025 * sr)
    dry, pos, h = so.synth_dry(rng, N), so.synth_path(rng, P), so.synth_rirs(rng, P, C, L)
    noise, music = so.synth_dry(rng, N), so.synth_dry(rng, N)
    hn, hm = so.synth_rirs(rng, 1, C, L)[0], so.synth_rirs(rng, 1, C, L)[0]
    np.random.seed(5001)
    bounds = render.trajectory_bounds(pos, N)
    out_d = np.empty((C, N), np.float32)
    outs = render.default_renderer().render_host(
        [render.MovingSource(dry, h, bounds, direct_taps=taps), render.StaticSource(noise, hn),
         render.StaticSource(music, hm)], direct_outs=[out_d, None, None])
    idx = np.repeat(np.arange(P - 1), np.diff(bounds))
    w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(bounds)]).astype(np.float32)
    assert so.rel_rms(outs[0], so.convolve_moving_receiver(dry, h, idx, w)) < TOL
    assert so.rel_rms(out_d, so.convolve_moving_receiver(dry, direct_path_rirs(h, taps), idx, w)) < TOL
    assert so.rel_rms(outs[1], so.convolve_fixed_receiver(noise[None], hn)) < TOL
    assert so.rel_rms(outs[2], so.convolve_fixed_receiver(music[None], hm)) < TOL


@pytest.mark.parametrize("name", ["bounds", "static2"])
def test_loudness_target_scales_the_direct_stem_by_the_reverberant_gain(name):
    from sonicsim_b200 import render
    R = render.default_renderer()
    x, h, idx, w, bounds, taps = make_case(name)
    dual = _sources(x, h, bounds, False, taps)[0]
    C, N = h.shape[1], x.shape[0]
    raw_d = np.empty((C, N), np.float32)
    raw = R.render_host([dual], direct_outs=[raw_d])[0]
    norm_d = np.empty((C, N), np.float32)
    loud = []
    norm = R.render_host([dual], lufs_targets=[-23.0], loudness_out=loud, direct_outs=[norm_d])[0]
    gain = loud[0][1]
    assert np.isfinite(gain) and gain != 1.0
    assert np.array_equal(norm, raw * np.float32(gain))
    assert np.array_equal(norm_d, raw_d * np.float32(gain))


def test_invalid_direct_target_arguments():
    from sonicsim_b200 import _lib, render
    R = render.default_renderer()
    x, h, idx, w, bounds, taps = make_case("indexed")
    C, N = h.shape[1], x.shape[0]
    out, out_d = np.zeros((C, N), np.float32), np.zeros((C, N), np.float32)
    flag = _lib.SS_DIRECT_TARGET
    bad = [_indexed_item(x, h, idx, w, out, flag, None, taps),       # no out_direct
           _indexed_item(x, h, idx, w, out, flag, out_d, 0),         # direct_taps = 0
           _indexed_item(x, h, idx, w, out, flag, out, taps)]        # out_direct == out
    for it in bad:
        one = (_lib.SsSource * 1)(it)
        assert R.lib.ss_render_host(R.ctx, one, 1) == _lib.SS_ERR_INVALID
        assert R.lib.ss_render_dev(R.ctx, one, 1, None) == _lib.SS_ERR_INVALID
        plan = ctypes.c_void_p()
        assert R.lib.ss_plan_create(R.ctx, one, 1, ctypes.byref(plan)) == _lib.SS_ERR_INVALID
    good = (_lib.SsSource * 1)(_indexed_item(x, h, idx, w, out, flag, out_d, taps))
    assert R.lib.ss_render_host(R.ctx, good, 1) == _lib.SS_OK
    # the Python layer: a direct target needs its output, an output needs a direct target
    xb, hb, _, _, bb, tb = make_case("bounds")
    src = render.MovingSource(xb, hb, bb, direct_taps=tb)
    with pytest.raises(ValueError):
        R.render_host([src])
    with pytest.raises(ValueError):
        R.render_host([src], direct_outs=[None])
    with pytest.raises(ValueError):
        R.render_host([src._replace(direct_taps=0)], direct_outs=[np.empty((hb.shape[1], xb.shape[0]), np.float32)])
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    dsrc = render.MovingSource(to(xb), to(hb), to(bb), bb, False, tb)
    with pytest.raises(ValueError):
        R.plan_device([dsrc], [torch.empty((hb.shape[1], xb.shape[0]), device="cuda")])
    with pytest.raises(ValueError):
        R.render_device([dsrc], [torch.empty((hb.shape[1], xb.shape[0]), device="cuda")])
