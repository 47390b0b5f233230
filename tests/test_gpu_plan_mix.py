"""Mixtures in device plans (ss_plan_create_mix; Python: Renderer.plan_device(..., mixtures=[Mixture(...)])) through the
real kernels.  Every plan mixture must equal, bit for bit, ss_mix_dev run on copies of the plan's own stems with the same
SIR and SNR values, and through it tests/mix_reference.py: gains within 3 float32 ulps of the float64 gains, outputs the
exact float32 composition with those gains.  Outputs are NaN-filled views of buffers with sentinels on both sides.
Covers whole stems, fixed and moving windows, raw and banked RIRs, direct targets, shared noise stems, many runs with
starts, SIRs and SNRs rewritten on the stream, the channel-mean (mono) fold, silent crops, the graph and its launch
count, SS_NO_GRAPH and profiling runs, and the argument checks."""
import ctypes
import os

import numpy as np
import pytest
import torch

from mix_reference import F32, _rms_db, compose_mix, mix_gains_f64
from gpu_plumbing import renderer
from mix_reference import Mix, check_mix, fold, mix_dev

pytestmark = pytest.mark.gpu

SENT = 1234.5
PAD = 32                # floats: a view at PAD is 16-byte aligned (the float4 path), at PAD + off it is not
SR = 16000
SS_ERR_INVALID, SS_ERR_UNSUPPORTED = -1, -5


class Guarded:
    """A float32 tensor of `shape`, a NaN-filled view into a buffer with SENT on both sides."""

    def __init__(self, shape, off=0):
        self.shape, self.lo = tuple(shape), PAD + off
        n = int(np.prod(self.shape))
        self.buf = torch.full((n + self.lo + PAD,), float("nan"), device="cuda")
        self.buf[:self.lo] = SENT
        self.buf[-PAD:] = SENT
        self.t = self.buf[self.lo:self.lo + n].view(self.shape)

    def get(self, snap=None):
        a = (self.buf if snap is None else snap).cpu().numpy()
        assert np.all(a[:self.lo] == SENT) and np.all(a[-PAD:] == SENT), "sentinel overwritten"
        v = a[self.lo:-PAD].reshape(self.shape)
        assert not np.isnan(v).any(), "output not written"
        return v


def _bounds(N, P):
    return np.linspace(0, N, P).astype(np.int32)


class Stems:
    """The plan's sources and guarded outputs.  kind: "whole", "fixed" or "moving" (a device start per scene);
    speakers are moving sources (P = 4), noises static; `banked`: every RIR set through a RirBank; `direct`: speakers
    also render a direct-path stem."""

    def __init__(self, rng, kind, banked=False, direct=False, C=2, N=48000, T=16000, L=900):
        from oracle import sonicsim_oracle as so
        from sonicsim_b200 import render
        self.R, self.rng, self.kind, self.banked, self.direct = renderer(), rng, kind, banked, direct
        self.C, self.N, self.L = C, N, L
        self.T = N if kind == "whole" else T
        self.so, self.render = so, render
        self.sources, self.outs, self.douts, self.banks = [], [], [], []
        self.starts = torch.zeros(64, dtype=torch.int32, device="cuda")

    def _window(self, scene):
        if self.kind == "whole":
            return None
        if self.kind == "fixed":
            return (int(self.rng.integers(0, self.N - self.T + 1)), self.T)
        return (self.starts[scene], self.T)

    def _rir(self, h):
        if not self.banked:
            return torch.from_numpy(h).cuda()
        b = self.R.rir_bank(torch.from_numpy(h).cuda(), direct_taps=40 if self.direct else 0)
        self.banks.append(b)
        return b

    def add(self, scene, speaker, dry=None):
        so, render = self.so, self.render
        x = so.synth_dry(self.rng, self.N) if dry is None else dry
        win = self._window(scene)
        if speaker:
            h = so.synth_rirs(self.rng, 4, self.C, self.L)
            b = _bounds(self.N, 4)
            s = render.MovingSource(torch.from_numpy(x).cuda(), self._rir(h), torch.from_numpy(b).cuda(), b,
                                    direct_taps=40 if self.direct else 0, window=win)
        else:
            h = so.synth_rirs(self.rng, 1, self.C, self.L)[0] * F32(0.3)
            s = render.StaticSource(torch.from_numpy(x).cuda(), self._rir(h), window=win)
        self.sources.append(s)
        self.outs.append(torch.full((self.C, self.T), float("nan"), device="cuda"))
        self.douts.append(torch.full((self.C, self.T), float("nan"), device="cuda") if speaker and self.direct
                          else None)
        return len(self.sources) - 1

    def draw_starts(self):
        self.starts.copy_(torch.randint(0, self.N - self.T + 1, (64,), dtype=torch.int32, device="cuda"))

    def plan(self, mixtures=None):
        return self.R.plan_device(self.sources, self.outs, self.douts if self.direct else None, mixtures)

    def stem(self, i, mono=False):
        """Output i as the plan left it, flattened: (C * T,), or its channel mean folded in NumPy (float32 sum in
        channel order, then a division by C) with `mono`."""
        a = self.outs[i].cpu().numpy()
        assert not np.isnan(a).any()
        return fold(a) if mono else a.reshape(-1)

    def close(self):
        for b in self.banks:
            b.close()


class Scene:
    """One Mixture of the plan over guarded outputs, with its SIR / SNR tensors."""

    def __init__(self, stems, spk, noi, delay=0, mono=False, with_out=True, with_rms=True, sirs=None, snr=None, off=0):
        from sonicsim_b200 import render
        self.st, self.spk, self.noi, self.delay, self.mono = stems, spk, noi, delay, mono
        S = len(spk)
        row = (stems.T,) if mono else (stems.C, stems.T)
        self.g_mix = Guarded(row, off)
        self.g_out = Guarded((S,) + row, off) if with_out else None
        self.g_rms = Guarded((S,)) if with_rms else None
        self.sirs = torch.tensor(np.asarray(sirs if sirs is not None else stems.rng.uniform(-6, 6, S - 1), np.float32),
                                 device="cuda") if S > 1 else None
        self.snr = torch.tensor([snr if snr is not None else stems.rng.uniform(10, 20)], dtype=torch.float32,
                                device="cuda")
        self.m = render.Mixture(spk, noi, self.sirs, self.snr[0], self.g_mix.t,
                                self.g_out.t if self.g_out else None, self.g_rms.t if self.g_rms else None, mono,
                                delay)

    def twin(self):
        """ss_mix_dev on copies of the plan's stems, stacked into (S, E) and (M, E), with the same SIRs and SNR."""
        spk = np.stack([self.st.stem(i, self.mono) for i in self.spk])
        noi = np.stack([self.st.stem(i, self.mono) for i in self.noi])
        sirs = self.sirs.cpu().numpy() if self.sirs is not None else np.zeros(0, F32)
        c = Mix(spk, noi, sirs, float(self.snr.cpu()[0]), self.delay, "sep")
        assert mix_dev([c]) == 0
        return c

    def check(self):
        """The plan's outputs against its ss_mix_dev twin (bit for bit) and the float64 references; returns the twin
        and the recovered gains."""
        c = self.twin()
        tmix, tout = c.outputs()
        mix = self.g_mix.get().reshape(-1)
        assert np.array_equal(mix, tmix)
        if self.g_out is not None:
            assert np.array_equal(self.g_out.get().reshape(len(self.spk), -1), tout)
        if self.g_rms is not None:
            rms = self.g_rms.get()
            for s in range(len(self.spk)):
                assert abs(float(rms[s]) - _rms_db(c.spk[s])) <= 1e-6, (s, rms[s], _rms_db(c.spk[s]))
        return c, check_mix(c, tmix, tout)


CASES = {  # kind, banked, direct, S, M, noise_delay
    "whole-raw-s1m1": ("whole", False, False, 1, 1, 0),
    "whole-bank-s2m2-delay": ("whole", True, False, 2, 2, SR),
    "fixed-raw-s3m1": ("fixed", False, False, 3, 1, 0),
    "fixed-bank-s2m2-delay": ("fixed", True, False, 2, 2, SR),
    "moving-bank-s2m1": ("moving", True, False, 2, 1, 0),
    "moving-raw-s3m2-delay": ("moving", False, False, 3, 2, SR),
    "moving-bank-direct-s2m1-delay": ("moving", True, True, 2, 1, SR),
    "fixed-raw-direct-s1m2": ("fixed", False, True, 1, 2, 0),
}


@pytest.mark.parametrize("name", list(CASES))
def test_plan_mixture_equals_mix_dev(name):
    """Two scenes in one plan, the second sharing the first's noise stems; both mixtures equal ss_mix_dev on their
    stems bit for bit, and the plan's direct stems are still rendered."""
    kind, banked, direct, S, M, delay = CASES[name]
    rng = np.random.default_rng(list(CASES).index(name))
    st = Stems(rng, kind, banked, direct)
    spk0 = [st.add(0, True) for _ in range(S)]
    noi = [st.add(0, False) for _ in range(M)]
    spk1 = [st.add(1 if kind == "moving" else 0, True) for _ in range(S)]
    scenes = [Scene(st, spk0, noi, delay), Scene(st, spk1, noi, delay, with_out=S > 1, with_rms=False)]
    st.draw_starts()
    plan = st.plan([s.m for s in scenes])
    plan.run()
    torch.cuda.synchronize()
    for s in scenes:
        s.check()
    if direct:
        for d in st.douts:
            if d is not None:
                assert not torch.isnan(d).any()
    plan.close()
    st.close()


def test_many_runs_without_host_synchronise():
    """8 scenes of 2 speakers and 1 static noise, 4 s crops, the stems of a scene sharing one start element.  Starts,
    SIRs and SNRs are rewritten on the stream with torch's RNG between runs and the outputs snapshotted on the stream;
    at the end every snapshot is ss_mix_dev of that run's crops (slices of the full stems) and the composition with
    gains within 3 ulps of the float64 gains.  The same inputs again give the same bits."""
    from sonicsim_b200 import render
    B, T, N, C = 8, 4 * SR, 5 * SR, 2
    rng = np.random.default_rng(3)
    st = Stems(rng, "moving", banked=True, C=C, N=N, T=T, L=2000)
    sc = [([st.add(b, True), st.add(b, True)], [st.add(b, False)]) for b in range(B)]
    mix, out, rms = Guarded((B, C, T)), Guarded((B, 2, C, T)), Guarded((B, 2))
    sirs = torch.zeros((B, 1), device="cuda")
    snr = torch.zeros((B,), device="cuda")
    mixtures = [render.Mixture(s, n, sirs[b], snr[b], mix.t[b], out.t[b], rms.t[b]) for b, (s, n) in enumerate(sc)]
    plan = st.plan(mixtures)
    full = [torch.empty((C, N), device="cuda") for _ in st.sources]
    st.R.render_device([s._replace(window=None) for s in st.sources], full)
    g = torch.Generator(device="cuda")
    g.manual_seed(11)
    snaps = []
    for _ in range(6):
        st.starts[:B].copy_(torch.randint(0, N - T + 1, (B,), dtype=torch.int32, device="cuda", generator=g))
        sirs.uniform_(-6, 6, generator=g)
        snr.uniform_(10, 20, generator=g)
        plan.run()
        snaps.append([x.clone() for x in (st.starts[:B], sirs, snr, mix.buf, out.buf, rms.buf)])
    torch.cuda.synchronize()
    assert plan.is_graph()
    fulls = [f.cpu().numpy() for f in full]
    for starts, s_sirs, s_snr, m_buf, o_buf, r_buf in snaps:
        a, sr_, sn_ = starts.cpu().numpy(), s_sirs.cpu().numpy(), s_snr.cpu().numpy()
        m_all, o_all, r_all = mix.get(m_buf), out.get(o_buf), rms.get(r_buf)
        for b, (s, n) in enumerate(sc):
            crop = lambda i: fulls[i][:, a[b]:a[b] + T].reshape(-1)              # noqa: E731
            c = Mix(np.stack([crop(i) for i in s]), np.stack([crop(i) for i in n]), sr_[b], float(sn_[b]), 0, "sep")
            assert mix_dev([c]) == 0
            tmix, tout = c.outputs()
            assert np.array_equal(m_all[b].reshape(-1), tmix) and np.array_equal(o_all[b].reshape(2, -1), tout)
            check_mix(c, tmix, tout)
            for k in range(2):
                assert abs(float(r_all[b, k]) - _rms_db(c.spk[k])) <= 1e-6
    # the first run's inputs again: the same bits
    starts, s_sirs, s_snr, m_buf, o_buf, _ = snaps[0]
    st.starts[:B].copy_(starts)
    sirs.copy_(s_sirs)
    snr.copy_(s_snr)
    plan.run()
    torch.cuda.synchronize()
    assert torch.equal(mix.buf, m_buf) and torch.equal(out.buf, o_buf)
    st.R.check_device_errors()
    plan.close()
    st.close()


@pytest.mark.parametrize("C", [1, 2, 5, 6, 8])
def test_mono_fold(C):
    """SS_MIX_MONO: bit for bit ss_mix_dev on the stems folded in NumPy (float32 channel sum in order, then / C), on
    the float4 path (T a multiple of 4, aligned outputs) and the scalar path (the same mixture into outputs one float
    off alignment - identical bits -, odd T, and a shifted noise).  Against the dataloader
    computed with torch's own x.mean(dim=0): every folded element within C float32 ulps of its channels' mean
    magnitude (speaker 0's scaled stem is its fold, gain 1), and every mixture element within 16 ulps of the magnitude
    it is built from."""
    rng = np.random.default_rng(C)
    for T, delay in ((16000, 0), (15999, 0), (16000, 7)):
        st = Stems(rng, "fixed", banked=True, C=C, T=T)
        spk, noi = [st.add(0, True), st.add(0, True)], [st.add(0, False), st.add(0, False)]
        scene = Scene(st, spk, noi, delay, mono=True)
        shifted = Scene(st, spk, noi, delay, mono=True, sirs=scene.sirs.cpu().numpy(), snr=float(scene.snr[0]), off=1)
        plan = st.plan([scene.m, shifted.m])
        plan.run()
        torch.cuda.synchronize()
        _, (g, gn) = scene.check()
        shifted.check()
        assert np.array_equal(scene.g_mix.get(), shifted.g_mix.get())
        assert np.array_equal(scene.g_out.get(), shifted.g_out.get())
        # torch's mean against the fold
        raw = [torch.from_numpy(st.outs[i].cpu().numpy()) for i in spk + noi]
        tm = [r.mean(dim=0).numpy() for r in raw]
        scale = [np.abs(r.numpy()).mean(axis=0).astype(np.float64) for r in raw]
        ulp = 2.0 ** -23
        fold0 = scene.g_out.get()[0]
        assert np.all(np.abs(fold0.astype(np.float64) - tm[0]) <= C * ulp * scale[0] + 1e-45)
        ref = compose_mix(np.stack(tm[:2]), np.stack(tm[2:]), g, gn, delay)[0]
        mag = g[0] * scale[0] + g[1] * scale[1] + gn * (scale[2] + scale[3]) * (3 if delay else 1)
        assert np.all(np.abs(scene.g_mix.get().astype(np.float64) - ref) <= 16 * ulp * mag + 1e-45)
        plan.close()
        st.close()


def test_silent_speaker_crop():
    """A speaker whose crop lies in a silent stretch of its dry signal: rms_db = -200 (the 1e-20 floor); the
    interferer's gain clamps at +40 dB (exactly 100.0f) and the mixture is still the reference arithmetic."""
    from sonicsim_b200 import render
    rng = np.random.default_rng(9)
    N, T, C = 80000, 16000, 2
    st = Stems(rng, "fixed", C=C, N=N, T=T, L=900)
    x = st.so.synth_dry(rng, N)
    x[16384:65536] = 0
    # static speakers: grid blocking, so every block that meets the crop (and its transform partner) reads silence
    for scene, dry in ((0, None), (0, x)):
        xx = st.so.synth_dry(rng, N) if dry is None else dry
        h = st.so.synth_rirs(rng, 1, C, 900)[0]
        st.sources.append(render.StaticSource(torch.from_numpy(xx).cuda(), torch.from_numpy(h).cuda(),
                                              window=(28672, T)))
        st.outs.append(torch.full((C, T), float("nan"), device="cuda"))
        st.douts.append(None)
    noi = st.add(0, False)
    scene = Scene(st, [0, 1], [noi], sirs=[0.0], snr=15.0)
    plan = st.plan([scene.m])
    plan.run()
    torch.cuda.synchronize()
    assert not st.outs[1].any()
    rms = scene.g_rms.get()
    assert rms[1] == F32(-200.0) and rms[0] > -60
    c, _ = scene.check()                 # the outputs are compose_mix of gains within 3 ulps of the float64 gains ...
    g64, _ = mix_gains_f64(c.spk, c.noise, c.sirs, c.snr)
    assert g64[1] == 100.0                # ... whose interferer gain is clamped at +40 dB
    assert not scene.g_out.get()[1].any() and np.all(np.isfinite(scene.g_mix.get()))
    plan.close()


def _graph_case():
    rng = np.random.default_rng(21)
    st = Stems(rng, "moving", banked=False, C=2)
    scenes = []
    for b in range(2):
        s, n = [st.add(b, True), st.add(b, True)], [st.add(b, False)]
        scenes.append(Scene(st, s, n, mono=b == 1))
    st.draw_starts()
    return st, scenes


def _bits(st, scenes):
    torch.cuda.synchronize()
    return [o.cpu().numpy().copy() for o in st.outs] + [x.buf.cpu().numpy().copy() for s in scenes
                                                        for x in (s.g_mix, s.g_out, s.g_rms)]


def _same(a, b):
    assert len(a) == len(b) and all(np.array_equal(x, y, equal_nan=True) for x, y in zip(a, b))


def test_graph_launches_no_graph_and_profiling():
    from sonicsim_b200 import _lib as L
    st, scenes = _graph_case()
    R = st.R
    plan = st.plan([s.m for s in scenes])
    plan.run()
    ref = _bits(st, scenes)
    for s in scenes:
        s.check()
    assert plan.is_graph()
    c0 = R.launch_count()
    plan.run()
    with_mix = R.launch_count() - c0
    _same(ref, _bits(st, scenes))
    bare = st.plan()                                                    # ss_plan_create on the same items
    c0 = R.launch_count()
    bare.run()
    without = R.launch_count() - c0
    assert with_mix == without + 4
    stems = _bits(st, [])
    # mixtures=None / [] in Python, and ss_plan_create_mix with n_mixes = 0: ss_plan_create's launches and bits
    for p in (st.plan(None), st.plan([])):
        c0 = R.launch_count()
        p.run()
        assert R.launch_count() - c0 == without
        _same(stems, _bits(st, []))
        p.close()
    items, n, _ = R._device_items(st.sources, st.outs)
    h = ctypes.c_void_p()
    L.check(R.lib.ss_plan_create_mix(R.ctx, items, n, None, 0, ctypes.byref(h)))
    for o in st.outs:
        o.fill_(float("nan"))
    c0 = R.launch_count()
    L.check(R.lib.ss_plan_run(h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert R.launch_count() - c0 == without
    _same(stems, _bits(st, []))
    R.lib.ss_plan_destroy(h)
    # profiling runs: the same bits
    for s in scenes:
        for x in (s.g_mix, s.g_out, s.g_rms):
            x.t.fill_(float("nan"))
    R.set_profiling(True)
    try:
        plan.run()
        R.get_profile()
    finally:
        R.set_profiling(False)
    _same(ref, _bits(st, scenes))
    # SS_NO_GRAPH: a context created with it set enqueues the launches; the same bits
    os.environ["SS_NO_GRAPH"] = "1"
    ctx2 = ctypes.c_void_p()
    try:
        L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
    finally:
        del os.environ["SS_NO_GRAPH"]
    for s in scenes:
        for x in (s.g_mix, s.g_out, s.g_rms):
            x.t.fill_(float("nan"))
    items, n, keep = R._device_items(st.sources, st.outs)
    mixes = R._device_mixes([s.m for s in scenes], st.outs, keep)
    h = ctypes.c_void_p()
    L.check(R.lib.ss_plan_create_mix(ctx2, items, n, mixes, len(mixes), ctypes.byref(h)))
    L.check(R.lib.ss_plan_run(h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    assert R.lib.ss_plan_is_graph(h) == 0
    _same(ref, _bits(st, scenes))
    R.lib.ss_plan_destroy(h)
    R.lib.ss_destroy(ctx2)
    plan.close()
    bare.close()


# ---- argument checks
def test_c_abi_refusals():
    """Every refusal returns its status, creates no plan and writes nothing: all outputs live in one NaN arena."""
    from sonicsim_b200 import _lib as L
    st, scenes = _graph_case()
    R = st.R
    items, n, keep = R._device_items(st.sources, st.outs)
    E = st.C * st.T
    arena = torch.full((8 * E + 64,), float("nan"), device="cuda")
    at = lambda i: arena.data_ptr() + 4 * i                      # noqa: E731
    sirs = torch.tensor([1.0, 2.0], device="cuda")
    base = [dict(speakers=(0, 1), noises=(2,), S=2, M=1, sirs=sirs.data_ptr(), snr=sirs.data_ptr() + 4,
                 mix=at(0), speakers_out=at(E), rms_db=at(3 * E), flags=0, noise_delay=0),
            dict(speakers=(3, 4), noises=(5,), S=2, M=1, sirs=sirs.data_ptr(), snr=sirs.data_ptr() + 4,
                 mix=at(4 * E), speakers_out=None, rms_db=None, flags=L.SS_MIX_MONO, noise_delay=3)]

    def arr(mods=({}, {}), count=None):
        out = []
        for b, mod in zip(base, mods):
            d = {**b, **mod}
            e = L.SsPlanMix()
            for i, v in enumerate(d.pop("speakers")):
                e.speakers[i] = v
            for i, v in enumerate(d.pop("noises")):
                e.noises[i] = v
            for k, v in d.items():
                setattr(e, k, v)
            out.append(e)
        if count:
            out = [out[0]] * count
        return (L.SsPlanMix * len(out))(*out)

    def create(a, n_items=n, its=items):
        h = ctypes.c_void_p()
        st_ = R.lib.ss_plan_create_mix(R.ctx, its, n_items, a, len(a), ctypes.byref(h))
        return st_, h

    before = arena.cpu().numpy()
    x0 = st.sources[0].dry.data_ptr()
    bad = [  # (status, mixture 0 changes, mixture 1 changes)
        (SS_ERR_INVALID, {"speakers": (0, n)}, {}),
        (SS_ERR_INVALID, {"noises": (-1,)}, {}),
        (SS_ERR_INVALID, {"speakers": (0, 0)}, {}),
        (SS_ERR_INVALID, {"noises": (1,)}, {}),                                 # a speaker is also a noise
        (SS_ERR_UNSUPPORTED, {"S": 0}, {}),
        (SS_ERR_UNSUPPORTED, {"S": 9}, {}),
        (SS_ERR_UNSUPPORTED, {"M": 0}, {}),
        (SS_ERR_UNSUPPORTED, {"M": 9}, {}),
        (SS_ERR_INVALID, {"snr": None}, {}),
        (SS_ERR_INVALID, {"sirs": None}, {}),
        (SS_ERR_INVALID, {"mix": None}, {}),
        (SS_ERR_INVALID, {"flags": 2}, {}),
        (SS_ERR_INVALID, {"noise_delay": -1}, {}),
        (SS_ERR_INVALID, {"mix": at(E + 5)}, {}),                               # mix inside its speakers_out
        (SS_ERR_INVALID, {"rms_db": at(E - 1)}, {}),                            # rms_db meets its own mix
        (SS_ERR_INVALID, {}, {"mix": at(3 * E + 1)}),                           # another mixture's rms_db
        (SS_ERR_INVALID, {}, {"mix": at(2 * E)}),                               # another mixture's speakers_out
        (SS_ERR_INVALID, {"mix": sirs.data_ptr() + 4}, {}),                     # a mixture's snr
        (SS_ERR_INVALID, {}, {"rms_db": sirs.data_ptr() - 4}),                  # rms_db's second float on the sirs
        (SS_ERR_INVALID, {"speakers_out": st.outs[0].data_ptr()}, {}),          # on a stem
        (SS_ERR_INVALID, {"mix": st.outs[5].data_ptr() + 4 * (E - 1)}, {}),     # mix's first float is a stem's last
        (SS_ERR_INVALID, {"rms_db": x0 + 8}, {}),                               # inside an item's dry signal
        (SS_ERR_INVALID, {"mix": st.starts.data_ptr() - 4}, {}),                # meets a win_start_dev
    ]
    for status, m0, m1 in bad:
        got, h = create(arr((m0, m1)))
        assert got == status and not h.value, (status, m0, m1, got)
    assert create(arr(count=65536))[0] == SS_ERR_UNSUPPORTED
    # stems of one mixture that differ in C or T: a source rendering a shorter window, and one with more channels
    from sonicsim_b200 import render
    xtra = [st.sources[2]._replace(window=(0, st.T - 1)), st.sources[2]._replace(rir=torch.zeros(3, 10, device="cuda"))]
    xouts = [torch.full((st.C, st.T - 1), float("nan"), device="cuda"), torch.full((3, st.T), float("nan"), device="cuda")]
    its2, n2, _ = R._device_items(list(st.sources) + xtra, list(st.outs) + xouts)
    for j in (n, n + 1):
        got, h = create(arr(({"noises": (j,)}, {})), n2, its2)
        assert got == SS_ERR_INVALID and not h.value
    torch.cuda.synchronize()
    assert np.array_equal(arena.cpu().numpy(), before, equal_nan=True)
    assert all(torch.isnan(o).all() for o in st.outs)
    # the valid set is accepted and writes where it should
    got, h = create(arr())
    assert got == 0 and h.value
    L.check(R.lib.ss_plan_run(h, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    a = arena.cpu().numpy()
    assert np.all(np.isfinite(a[:3 * E + 2])) and np.all(np.isfinite(a[4 * E:4 * E + st.T]))
    R.lib.ss_plan_destroy(h)


def test_python_refusals():
    from sonicsim_b200 import render
    st, scenes = _graph_case()
    m = scenes[0].m
    E = (st.C, st.T)
    bad = [m._replace(mix=torch.zeros(E, dtype=torch.float64, device="cuda")),           # dtype
           m._replace(mix=torch.zeros(E)),                                               # device
           m._replace(mix=torch.zeros((st.C, st.T + 1), device="cuda")),                 # shape
           m._replace(mix=torch.zeros((st.T, st.C), device="cuda").t()),                 # not contiguous
           m._replace(speakers_out=torch.zeros((3,) + E, device="cuda")),                # shape
           m._replace(rms_db=torch.zeros(3, device="cuda")),                             # shape
           m._replace(sirs=torch.zeros(2, device="cuda")),                               # element count
           m._replace(sirs=None),                                                        # missing with S = 2
           m._replace(snr=torch.zeros(2, device="cuda")),                                # element count
           m._replace(snr=torch.zeros(1, dtype=torch.float64, device="cuda")),           # dtype
           m._replace(speakers=[0, 99]),                                                 # index
           m._replace(noises=[0]),                                                       # repeated
           m._replace(noises=[]),                                                        # M = 0
           m._replace(noise_delay=-1),
           m._replace(mono=True)]                                                        # mix is (C, T), not (T,)
    for b in bad:
        with pytest.raises(ValueError):
            st.plan([b])
    with pytest.raises(ValueError):                                                      # S = 1 takes no sirs
        st.plan([m._replace(speakers=[0], speakers_out=None, rms_db=None)])
    # outputs meeting each other are refused by the library, also as ValueError
    with pytest.raises(ValueError):
        st.plan([m, m])
    with pytest.raises(ValueError):
        st.plan([m._replace(mix=st.outs[5])])
    assert isinstance(render.Mixture([0], [1], None, scenes[0].snr[0], scenes[0].g_mix.t), render.Mixture)
