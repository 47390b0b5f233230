"""Dereverberation targets of plan mixtures (ss_plan_create_target; Python: Mixture(..., direct_out=...)) through the real
kernels.  Target s of a mixture is fold(direct stem of speaker s) * g_s, with the fold, the float32 gain and the single
rounded multiply that give speakers_out[s] from the reverberant stem.
  1. exact oracle: over RIR sets cut at their whole length (direct_taps >= L), a direct stem has its reverberant stem's
     bits, so direct_out must equal speakers_out bit for bit - mono and channels, S = 1, 2, 3, 8, M = 1, 2, T a multiple
     of 4 and not, noise_delay 0 and > 0, an unaligned direct_out: both write paths;
  2. real cuts (direct_taps = 40) on pooled training plans, 16 examples x (2 speakers + noise), 4 s crops, CropDraws: a
     device pool with dry picks and pair gains, and a tap-form host pool with a 16-bit host dry pool.  For every speaker,
     direct_out[s] == fold_f32(direct stem) * gf_s exactly, gf_s the float32 gain that reproduces speakers_out[s] from
     the reverberant stem (searched within 3 ulps of the float64 gain); and against float64;
  3. the same plan with and without targets: the same bits everywhere else, the same launches per run, one graph;
  4. runs without a host synchronise, everything redrawn between runs, and a run on a side stream;
  5. refusals of the C ABI and of Python, which leave no plan."""
import ctypes

import numpy as np
import pytest
import torch

from mix_reference import F32, f32_neighbours, mix_gains_f64
from oracle import sonicsim_oracle as so
from gpu_plumbing import _R, to

pytestmark = pytest.mark.gpu

RATE = 16000
CROP = 4 * RATE
U = 16                      # examples per step: 2 speakers + 1 noise each
TRIES = 101
TAPS = 40
SS_ERR_INVALID = -1


def fold_f32(a):
    """(C, T) -> (T,): float32 sum of the rows in channel order, then a division by C (the kernels' fold)."""
    a = np.asarray(a, F32)
    acc = a[0].copy()
    for c in range(1, a.shape[0]):
        acc = acc + a[c]
    return acc / F32(a.shape[0])


def _row(a, mono):
    return fold_f32(a) if mono else np.asarray(a, F32).reshape(-1)


# ---- 1. exact oracle: direct sets equal to the full RIRs

EXACT = {  # S, M, mono, C, T, noise_delay, offset of direct_out in floats
    "s1m1-mono": (1, 1, True, 2, 8000, 0, 0),
    "s2m2-chan": (2, 2, False, 2, 8000, 0, 0),
    "s3m1-mono-odd-T": (3, 1, True, 3, 7999, 0, 0),
    "s8m2-chan-unaligned-target": (8, 2, False, 2, 8000, 0, 1),
    "s2m1-mono-delay": (2, 1, True, 2, 8000, 400, 0),
    "s3m2-c1-odd-E": (3, 2, False, 1, 8001, 0, 0),
    "s8m1-mono-c4": (8, 1, True, 4, 8000, 0, 0),
    "s2m2-chan-delay-unaligned": (2, 2, False, 2, 8000, 7, 3),
}


@pytest.mark.parametrize("name", list(EXACT))
def test_full_cut_targets_equal_speakers_out(name):
    """Two mixtures in one plan; the first has a target, the second none (null pointers in a k_mix_write<true> plan).
    The first's direct_out equals its speakers_out bit for bit; both mixtures equal the plan without targets."""
    render, R = _R()
    S, M, mono, C, T, delay, off = EXACT[name]
    rng = np.random.default_rng(list(EXACT).index(name) + 11)
    N, L, P = T + 3000, 700, 3
    sources, outs, douts = [], [], []

    def add(speaker):
        x = so.synth_dry(rng, N)
        start = int(rng.integers(0, N - T + 1))
        if speaker:
            b = np.linspace(0, N, P).astype(np.int32)
            s = render.MovingSource(to(x), to(so.synth_rirs(rng, P, C, L)), to(b), b, direct_taps=L, window=(start, T))
        else:
            s = render.StaticSource(to(x), to(so.synth_rirs(rng, 1, C, L)[0] * F32(0.3)), window=(start, T))
        sources.append(s)
        outs.append(torch.full((C, T), float("nan"), device="cuda"))
        douts.append(torch.full((C, T), float("nan"), device="cuda") if speaker else None)
        return len(sources) - 1

    row = (T,) if mono else (C, T)
    mixes = []
    for k in range(2):
        spk = [add(True) for _ in range(S)]
        noi = [add(False) for _ in range(M)]
        sirs = torch.tensor(rng.uniform(-6, 6, S - 1).astype(F32), device="cuda") if S > 1 else None
        snr = torch.tensor([rng.uniform(10, 20)], dtype=torch.float32, device="cuda")
        mixes.append((spk, noi, sirs, snr))

    def plan(targets):
        o = {"mix": [], "spk_out": [], "rms": []}
        ms = []
        n_dir = S * int(np.prod(row))
        buf = torch.full((n_dir + off,), float("nan"), device="cuda")
        o["dir"] = buf[off:].view((S,) + row)
        for k, (spk, noi, sirs, snr) in enumerate(mixes):
            o["mix"].append(torch.full(row, float("nan"), device="cuda"))
            o["spk_out"].append(torch.full((S,) + row, float("nan"), device="cuda"))
            o["rms"].append(torch.full((S,), float("nan"), device="cuda"))
            ms.append(render.Mixture(spk, noi, sirs, snr[0], o["mix"][-1], o["spk_out"][-1], o["rms"][-1], mono, delay,
                                     o["dir"] if targets and k == 0 else None))
        return R.plan_device(sources, outs, douts, ms), o

    p_t, o_t = plan(True)
    p_t.run()
    torch.cuda.synchronize()
    got = {k: [t.clone() for t in v] if isinstance(v, list) else v.clone() for k, v in o_t.items()}
    stems = [t.clone() for t in outs]
    dstems = [t.clone() for t in douts if t is not None]
    p_0, o_0 = plan(False)
    p_0.run()
    torch.cuda.synchronize()
    for a, b in zip(stems, outs):
        assert torch.equal(a, b)
    for a, b in zip(dstems, [t for t in douts if t is not None]):
        assert torch.equal(a, b)
    for i, d in enumerate(douts):
        if d is not None:
            assert torch.equal(d, outs[i]), "a full cut must give the reverberant stem's bits"
    for key in ("mix", "spk_out", "rms"):
        for a, b in zip(got[key], o_0[key]):
            assert not torch.isnan(a).any() and torch.equal(a, b), key
    assert torch.equal(got["dir"], got["spk_out"][0])
    p_t.close()
    p_0.close()


# ---- 2-4. pooled training plans with real cuts

class Cand:
    def __init__(self, rng, N, P, C, L):
        self.x = so.synth_dry(rng, N)
        self.x[int(rng.integers(0, N // 2)):][:int(rng.integers(0, N // 4))] = 0      # a silent stretch
        self.h = so.synth_rirs(rng, P, C, L) * F32(0.6)
        self.b = None if P == 1 else np.round(np.linspace(0, N, P)).astype(np.int32)
        self.P = P


def _grid(x):
    return np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.float32) / np.float32(32768.0)


@pytest.fixture(scope="module")
def world():
    """Per form, (speaker pool, noise pool, dry pool, pair gains or None): "device" - device pools, a device float dry
    pool with level tables and pair gains; "taps" - tap-form host pools and a 16-bit host dry pool with level tables."""
    render, R = _R()
    rng = np.random.default_rng(4242)
    spk = [Cand(rng, 80000 + 7001 * j, 3 + j % 3, 2, (2048, 3000)[j % 2]) for j in range(6)]
    noi = [Cand(rng, 70000 + 9001 * j, 1, 2, 2048) for j in range(3)]
    n_max = max(len(c.x) for c in spk + noi)
    sig = [_grid(so.synth_dry(rng, n_max + 64 * j)) for j in range(5)]
    forms = {}
    dev_spk = [render.MovingSource(to(c.x), R.rir_bank(to(c.h), direct_taps=TAPS), to(c.b), c.b) for c in spk]
    dev_noi = [render.StaticSource(to(c.x), R.rir_bank(to(c.h[0]))) for c in noi]
    dpool = R.dry_pool([to(s) for s in sig], levels=True)
    pool = R.source_pool(dev_spk)
    gains = R.pair_gains(pool, dpool, -18.0 - rng.random((len(sig), len(spk))), sr=RATE)
    forms["device"] = (pool, R.source_pool(dev_noi), dpool, gains)
    host_spk = [render.MovingSource(c.x, R.rir_bank(c.h, False, TAPS, host=True, form="taps"), c.b, c.b) for c in spk]
    host_noi = [render.StaticSource(c.x, R.rir_bank(c.h[0], host=True, form="taps")) for c in noi]
    forms["taps"] = (R.source_pool(host_spk), R.source_pool(host_noi),
                     R.dry_pool(sig, levels=True, host=True, dtype="int16"), None)
    return forms, len(spk), len(noi), len(sig)


class Inputs:
    def __init__(self):
        self.picks = torch.zeros((U, 3), dtype=torch.int32, device="cuda")
        self.dry_picks = torch.zeros((U, 2), dtype=torch.int32, device="cuda")
        self.u = torch.zeros((U, TRIES), dtype=torch.float64, device="cuda")
        self.sirs = torch.zeros((U, 1), device="cuda")
        self.snr = torch.zeros((U, 1), device="cuda")

    def choose(self, n_spk, n_noi, n_dry):
        """Everything a step draws, on the current stream."""
        self.picks[:, :2].copy_(torch.rand(U, n_spk, device="cuda").argsort(1)[:, :2].int())
        self.picks[:, 2].random_(0, n_noi)
        self.dry_picks.random_(0, n_dry)
        self.u.uniform_()
        self.sirs.uniform_(-6, 6)
        self.snr.uniform_(10, 20)


def _mono(b):
    return b % 2 == 0


def _delay(b):
    return 5 if b == 3 else 0                          # one example on the scalar write path


def _train_plan(render, R, form, inp, targets):
    spk, noi, dry, gains = form
    starts = torch.zeros(U, dtype=torch.int32, device="cuda")
    used = torch.zeros(U, dtype=torch.int32, device="cuda")
    o = {"out": [], "direct": [], "mix": [], "spk_out": [], "rms": [], "dir": [], "starts": starts, "used": used}
    sources, direct_outs, mixtures, draws = [], [], [], []
    for b in range(U):
        base = len(sources)
        for k in range(2):
            sources.append(render.Pooled(spk, inp.picks[b, k], (starts[b], CROP), TAPS,
                                         render.DryPick(dry, inp.dry_picks[b, k], gains)))
            o["out"].append(torch.zeros((2, CROP), device="cuda"))
            direct_outs.append(torch.zeros((2, CROP), device="cuda"))
            o["direct"].append(direct_outs[-1])
        sources.append(render.Pooled(noi, inp.picks[b, 2], (starts[b], CROP)))
        o["out"].append(torch.zeros((2, CROP), device="cuda"))
        direct_outs.append(None)
        shape = (CROP,) if _mono(b) else (2, CROP)
        o["mix"].append(torch.zeros(shape, device="cuda"))
        o["spk_out"].append(torch.zeros((2,) + shape, device="cuda"))
        o["rms"].append(torch.zeros(2, device="cuda"))
        o["dir"].append(torch.full((2,) + shape, float("nan"), device="cuda") if targets else None)
        mixtures.append(render.Mixture([base, base + 1], [base + 2], inp.sirs[b], inp.snr[b], o["mix"][-1],
                                       o["spk_out"][-1], o["rms"][-1], _mono(b), _delay(b), o["dir"][-1]))
        draws.append(render.CropDraw(starts[b], [base, base + 1], inp.u[b], used[b]))
    return R.plan_device(sources, o["out"], direct_outs=direct_outs, mixtures=mixtures, draws=draws), o


def _snap(o, inp):
    s = {k: [t.clone() for t in v if t is not None] if isinstance(v, list) else v.clone() for k, v in o.items()}
    s["sirs"], s["snr"] = inp.sirs.clone(), inp.snr.clone()
    return s


def _check_targets(s):
    """Item 2's checks on one snapshot (tensors still on the device)."""
    h = {k: [t.cpu().numpy() for t in v] if isinstance(v, list) else v.cpu().numpy() for k, v in s.items()}
    worst = 0.0
    for b in range(U):
        mono, delay = _mono(b), _delay(b)
        rev = np.stack([_row(h["out"][3 * b + k], mono) for k in range(2)])
        dirs = np.stack([_row(h["direct"][2 * b + k], mono) for k in range(2)])
        noise = _row(h["out"][3 * b + 2], mono)[None]
        sp_out = h["spk_out"][b].reshape(2, -1)
        tgt = h["dir"][b].reshape(2, -1)
        assert not np.isnan(tgt).any()
        assert np.array_equal(sp_out[0], rev[0]) and np.array_equal(tgt[0], dirs[0]), b      # speaker 0: gain 1
        g64, _ = mix_gains_f64(rev, noise, h["sirs"][b], h["snr"][b][0], delay)
        fits = [g for g in f32_neighbours(g64[1]) if np.array_equal(rev[1] * g, sp_out[1])]
        assert fits, ("speakers_out[1] is no float32 gain within 3 ulps times its stem", b, g64[1])
        assert any(np.array_equal(tgt[1], dirs[1] * g) for g in fits), b
        # against float64: the direct stems folded in float64, times the float64 gains
        C = 2
        for k in range(2):
            d = h["direct"][2 * b + k].astype(np.float64)
            f64 = d.mean(0) if mono else d.reshape(-1)
            mag = np.abs(d).mean(0) if mono else np.abs(f64)
            err = np.abs(tgt[k].astype(np.float64) - f64 * g64[k])
            bound = (C + 10) * 2.0 ** -24 * mag * g64[k]
            assert np.all(err <= bound), (b, k, float(np.max(err - bound)))
            worst = max(worst, float(np.max(err / np.maximum(mag * g64[k], 1e-30))))
    return worst


@pytest.mark.parametrize("name", ["device", "taps"])
def test_training_plan_targets(world, name):
    """Runs without a host synchronise and one on a side stream: every run's targets pass the exact and float64 checks;
    the same plan without targets gives the same bits everywhere else, with the same launches per run."""
    render, R = _R()
    forms, n_spk, n_noi, n_dry = world
    inp = Inputs()
    plan_t, o_t = _train_plan(render, R, forms[name], inp, True)
    plan_0, o_0 = _train_plan(render, R, forms[name], inp, False)
    torch.manual_seed(7)
    snaps = []
    for _ in range(4):
        inp.choose(n_spk, n_noi, n_dry)
        plan_t.run()
        snaps.append(_snap(o_t, inp))
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        inp.choose(n_spk, n_noi, n_dry)
        plan_t.run()
        snaps.append(_snap(o_t, inp))
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for s in snaps:
        _check_targets(s)
    # the same choices through the plan without targets: every other output keeps its bits
    counts = []
    for p in (plan_t, plan_0):
        R.reset_stats()
        p.run()
        counts.append(R.launch_count())
    torch.cuda.synchronize()
    assert counts[0] == counts[1]
    assert plan_t.is_graph() and plan_0.is_graph()
    for k in ("out", "direct", "mix", "spk_out", "rms"):
        for i, (a, b) in enumerate(zip(o_t[k], o_0[k])):
            assert torch.equal(a, b), (k, i)
    assert torch.equal(o_t["starts"], o_0["starts"]) and torch.equal(o_t["used"], o_0["used"])
    assert int(o_t["used"].min()) >= 0
    _check_targets(_snap(o_t, inp))
    R.check_device_errors()
    plan_t.close()
    plan_0.close()


# ---- 5. refusals

def test_refusals():
    render, R = _R()
    from sonicsim_b200 import _lib as L
    rng = np.random.default_rng(99)
    C, N, T, Lr = 2, 12000, 8000, 300
    sources, outs, douts = [], [], []
    for k in range(5):                                  # 0, 1: speakers with direct stems; 2: noise; 3, 4: no direct
        x = so.synth_dry(rng, N)
        h = so.synth_rirs(rng, 1, C, Lr)[0]
        direct = k < 2
        sources.append(render.StaticSource(to(x), to(h), direct_taps=TAPS if direct else 0, window=(100 * k, T)))
        outs.append(torch.zeros((C, T), device="cuda"))
        douts.append(torch.zeros((C, T), device="cuda") if direct else None)
    sirs, snr = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    mix0, mix1 = torch.zeros(T, device="cuda"), torch.zeros(T, device="cuda")
    sp0 = torch.zeros((2, T), device="cuda")
    tgt = torch.zeros((2, T), device="cuda")
    tgt2 = torch.zeros((2, T), device="cuda")
    M = [render.Mixture([0, 1], [2], sirs, snr[0], mix0, sp0, None, True),
         render.Mixture([3, 4], [2], sirs, snr[0], mix1, None, None, True)]
    items, n, keep = R._device_items(sources, outs, douts)
    mixes = R._device_mixes(M, outs, keep)

    def c_call(entries, n_targets=None, want=SS_ERR_INVALID):
        arr = (L.SsPlanTarget * max(1, len(entries)))(*[L.SsPlanTarget(mix=m, direct_out=p) for m, p in entries])
        h = ctypes.c_void_p()
        got = R.lib.ss_plan_create_target(R.ctx, items, n, mixes, 2, None, 0, None, None, 0, arr,
                                          len(entries) if n_targets is None else n_targets, ctypes.byref(h))
        assert got == want, (entries, got)
        if want == 0:
            assert h.value
            R.lib.ss_plan_destroy(h)
        else:
            assert h.value is None
    t, t2 = tgt.data_ptr(), tgt2.data_ptr()
    c_call([(0, t)], want=0)
    c_call([], want=0)                                   # no targets: ss_plan_create_pair
    c_call([(-1, t)])
    c_call([(2, t)])
    c_call([(0, t), (0, t2)])                            # a mixture named twice
    c_call([(0, None)])
    c_call([(1, t)])                                     # speakers 3, 4 render no direct stem
    c_call([(0, douts[0].data_ptr())])                   # over a direct stem the target reads
    c_call([(0, douts[1].data_ptr() - 4)])
    c_call([(0, mix0.data_ptr() + 4)])                   # over the mixture's own mix
    c_call([(0, sp0.data_ptr())])                        # over its speakers_out
    c_call([(0, outs[2].data_ptr())])                    # over a stem
    c_call([(0, sirs.data_ptr() - 4)])                   # over the sirs it reads
    c_call([(0, t)], n_targets=-1)
    h = ctypes.c_void_p()
    assert R.lib.ss_plan_create_target(R.ctx, items, n, mixes, 2, None, 0, None, None, 0, None, 1,
                                       ctypes.byref(h)) == SS_ERR_INVALID and h.value is None
    # two mixtures' targets over one range
    M2 = [M[0], render.Mixture([1, 0], [2], sirs, snr[0], mix1, None, None, True)]
    mixes2 = R._device_mixes(M2, outs, keep)
    arr = (L.SsPlanTarget * 2)(L.SsPlanTarget(mix=0, direct_out=t), L.SsPlanTarget(mix=1, direct_out=t + 4))
    assert R.lib.ss_plan_create_target(R.ctx, items, n, mixes2, 2, None, 0, None, None, 0, arr, 2,
                                       ctypes.byref(h)) == SS_ERR_INVALID and h.value is None

    # Python: checked before any C call
    def py(m, match):
        with pytest.raises(ValueError, match=match):
            R.plan_device(sources, outs, douts, [m])
    base = M[0]
    py(M[1]._replace(direct_out=tgt), "renders no direct-path stem")
    py(base._replace(direct_out=torch.zeros((2, T + 1), device="cuda")), "direct_out")
    py(base._replace(direct_out=torch.zeros((1, T), device="cuda")), "direct_out")
    py(base._replace(direct_out=torch.zeros((2, C, T), device="cuda")), "direct_out")
    py(base._replace(direct_out=torch.zeros((2, T), dtype=torch.float64, device="cuda")), "direct_out")
    py(base._replace(direct_out=torch.zeros((2, T))), "direct_out")
    py(base._replace(direct_out=torch.zeros((T, 2), device="cuda").t()), "direct_out")
    # and what the C ABI refuses surfaces as ValueError, with no plan: a target over the mixture's own speakers_out
    with pytest.raises(ValueError):
        R.plan_device(sources, outs, douts, [base._replace(direct_out=sp0)])
    plan = R.plan_device(sources, outs, douts, [base._replace(direct_out=tgt)])
    plan.run()
    torch.cuda.synchronize()
    assert torch.equal(tgt[0], fold_t(douts[0]))
    plan.close()


def fold_t(a):
    return torch.from_numpy(fold_f32(a.cpu().numpy())).cuda()
