"""Tap-form host banks (SS_BANK_TAPS, Renderer.rir_bank(host=True, form="taps")) through the real kernels: every candidate's
RIR taps in pinned host memory, k_stage copying each run's rows of taps and one k_prepare launch transforming them on the
device.  Every check compares against spectral host banks (form="spectra") of the same RIRs:
  1. banks: a tap bank holds no device memory, host_nbytes is 16384 * P * C * K plus the cut table, ss_bank_flags reports
     the flags; a whole-stem slot (every row staged) equals the spectral host pool and render_device over the device bank,
     bit for bit, unnormalised, normalised (nonzero taps: k_bank_taps divides) and normalised over an all-zero RIR set;
  2. bit identity: the training plan of test_gpu_host_pool.py - pooled speakers with direct targets in a mixed-L pool of
     normalised banks (abs-max 0.6: every stored tap divided on the device) with loudness gains, static noise and music
     pools, CropDraws, Mixtures with mono and noise_delay, probe slots at every candidate's first and last start, one
     run out of range - and a dry-pick plan - speakers from a host float dry pool with pair gains, music from a 16-bit
     dry pool - give the same outputs, starts, `used` and error bits over 24 runs;
  3. builds: level tables, loudness and pair gains equal the spectral pools', over the normalised speaker banks;
  4. launches: one kernel more per run than the spectral host-pool plan, as one graph launch; a side stream gives the
     same bits;
  5. device memory: building a tap-form host pool with level tables grows device memory by a bounded amount;
  6. refusals of SS_BANK_TAPS without SS_BANK_HOST, of pools that mix forms and of tap banks outside pools, in Python
     and the C ABI.
The tests hold well under 2 GB of pinned host memory."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from gpu_plumbing import _R, _errors, to

pytestmark = pytest.mark.gpu

RATE = 16000
LEN = 2 * RATE
TRIES = 101
TAPS = 40
FORMS = ("spectra", "taps")


class Cand:
    def __init__(self, rng, N, P, C, L):
        self.x = so.synth_dry(rng, N)
        self.x[int(rng.integers(0, N // 2)):][:int(rng.integers(0, N // 3))] = 0      # a silent stretch
        self.h = so.synth_rirs(rng, P, C, L) * np.float32(0.6)
        self.b = None if P == 1 else np.round(np.linspace(0, N, P)).astype(np.int32)
        self.N, self.P, self.C, self.L = N, P, C, L


def _sources(R, render, cands, form, taps=0, normalize=False):
    out = []
    for c in cands:
        bank = R.rir_bank(c.h if c.P > 1 else c.h[0], normalize, taps, host=True, form=form)
        out.append(render.StaticSource(c.x, bank) if c.P == 1 else render.MovingSource(c.x, bank, c.b))
    return out


def _pool(R, render, cands, form, taps=0, levels=None, lufs=None, normalize=False):
    return R.source_pool(_sources(R, render, cands, form, taps, normalize), levels=levels, lufs_targets=lufs, sr=RATE)


def _grid(x):
    return np.clip(np.round(x * 32768.0), -32768, 32767).astype(np.float32) / np.float32(32768.0)


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    rng = np.random.default_rng(2027)
    spk = [Cand(rng, 120000 + 9001 * j, 3 + j % 4, 2, (4096, 9000, 3000)[j % 3]) for j in range(7)]
    noi = [Cand(rng, 100000 + 13007 * j, 1, 2, (4096, 6000)[j % 2]) for j in range(4)]
    mus = [Cand(rng, 90000 + 7919 * j, 1, 2, 2048) for j in range(3)]
    n_max = max(c.N for c in spk + noi + mus)
    sig = [so.synth_dry(rng, n_max + 50 * j) for j in range(5)]
    dry = {"host": R.dry_pool(sig, levels=True, host=True), "i16": R.dry_pool([_grid(s) for s in sig], dtype="int16")}
    targets = -18.0 - rng.random((len(sig), len(spk)))
    pools, gains = {}, {}
    for form in FORMS:
        pools[form] = (
            _pool(R, render, spk, form, TAPS, "mono", [-17.0 + 0.5 * j for j in range(len(spk))], normalize=True),
            _pool(R, render, noi, form, 0, None, [-24.0, None, -23.0, -25.0]),
            _pool(R, render, mus, form, 0, None, None))
        gains[form] = R.pair_gains(pools[form][0], dry["host"], targets, sr=RATE)
    return spk, noi, mus, pools, dry, gains


B = 3                                               # examples; each: 2 speakers, noise, music + 3 probe slots


class Inputs:
    def __init__(self):
        self.picks = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
        self.dry_picks = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
        self.probe_pick = torch.zeros(3, dtype=torch.int32, device="cuda")
        self.probe_start = torch.zeros(3, dtype=torch.int32, device="cuda")
        self.u = torch.zeros((B, TRIES), dtype=torch.float64, device="cuda")
        self.sirs = torch.zeros((B, 1), device="cuda")
        self.snr = torch.zeros((B, 1), device="cuda")


def _plan(render, R, pools, inp, dry=None, gains=None):
    """The training plan; with `dry` (the world's dry pools) the speakers are dry-picked from the host float dry pool
    with pair gains and the music slot from the 16-bit dry pool."""
    spk, noi, mus = pools
    starts = torch.zeros(B, dtype=torch.int32, device="cuda")
    used = torch.zeros(B, dtype=torch.int32, device="cuda")
    o = {"out": [], "direct": [], "mix": [], "spk_out": [], "rms": [], "starts": starts, "used": used}
    sources, direct_outs, mixtures, draws = [], [], [], []
    for b in range(B):
        base = len(sources)
        for k, pl in enumerate((spk, spk, noi, mus)):
            taps = TAPS if k < 2 else 0
            d = None
            if dry is not None and k < 2:
                d = render.DryPick(dry["host"], inp.dry_picks[b, k], gains)
            elif dry is not None and k == 3:
                d = render.DryPick(dry["i16"], inp.dry_picks[b, k])
            sources.append(render.Pooled(pl, inp.picks[b, k], (starts[b], LEN), taps, d))
            o["out"].append(torch.zeros((2, LEN), device="cuda"))
            direct_outs.append(torch.zeros((2, LEN), device="cuda") if taps else None)
        mono = b % 2 == 0
        shape = (LEN,) if mono else (2, LEN)
        o["mix"].append(torch.zeros(shape, device="cuda"))
        o["spk_out"].append(torch.zeros((2,) + shape, device="cuda"))
        o["rms"].append(torch.zeros(2, device="cuda"))
        mixtures.append(render.Mixture([base, base + 1], [base + 2, base + 3], inp.sirs[b], inp.snr[b], o["mix"][-1],
                                       o["spk_out"][-1], o["rms"][-1], mono, 0 if b == 1 else 3))
        draws.append(render.CropDraw(starts[b], [base, base + 1], inp.u[b], used[b]))
    for k, pl in enumerate((spk, noi, mus)):      # probes: starts written by the host, any candidate, any start
        sources.append(render.Pooled(pl, inp.probe_pick[k], (inp.probe_start[k], LEN), TAPS if k == 0 else 0))
        o["out"].append(torch.zeros((2, LEN), device="cuda"))
        direct_outs.append(torch.zeros((2, LEN), device="cuda") if k == 0 else None)
    o["direct"] = [d for d in direct_outs if d is not None]
    plan = R.plan_device(sources, o["out"], direct_outs=direct_outs, mixtures=mixtures, draws=draws)
    return plan, o


def _same(a, b, what):
    for k in ("out", "direct", "mix", "spk_out", "rms"):
        for i, (x, y) in enumerate(zip(a[k], b[k])):
            assert torch.equal(x, y), (what, k, i)
    assert torch.equal(a["starts"], b["starts"]) and torch.equal(a["used"], b["used"]), what


def test_pools_and_builds_equal(world):
    spk, noi, mus, pools, dry, gains = world
    for s, t in zip(pools["spectra"], pools["taps"]):
        assert s.resident == "host" and t.resident == "host"
        assert np.array_equal(s.loudness, t.loudness, equal_nan=True)
        assert s.nbytes == t.nbytes and s.host_nbytes == t.host_nbytes     # (banks not counted: same x and tables)
    s, t = pools["spectra"][0], pools["taps"][0]
    for i in range(s.n):
        assert torch.equal(s.level_table(i), t.level_table(i)), i
    assert np.array_equal(gains["spectra"].loudness, gains["taps"].loudness, equal_nan=True)


@pytest.mark.parametrize("dry_picks", [False, True], ids=["pooled", "dry_picked"])
def test_training_plan_bit_identity(world, dry_picks):
    render, R = _R()
    spk, noi, mus, pools, dry, gains = world
    inp = Inputs()
    args = lambda form: (dry, gains[form]) if dry_picks else (None, None)     # noqa: E731
    ps, os_ = _plan(render, R, pools["spectra"], inp, *args("spectra"))
    pt, ot = _plan(render, R, pools["taps"], inp, *args("taps"))
    rng = np.random.default_rng(8 + dry_picks)
    counts = (len(spk), len(spk), len(noi), len(mus))
    probes = [[(i, s) for i, c in enumerate(cs) for s in (0, c.N - LEN)] for cs in (spk, noi, mus)]
    runs = max(24, max(len(q) for q in probes) + 2)
    R.check_device_errors()
    for r in range(runs):
        picks = np.array([[rng.integers(0, n) for n in counts] for _ in range(B)], np.int32)
        inp.picks.copy_(torch.from_numpy(picks))
        inp.dry_picks.copy_(torch.from_numpy(rng.integers(0, 5, (B, 4)).astype(np.int32)))
        u = rng.random((B, TRIES))
        if r % 5 == 1:
            u[:] = 0.0                               # the first start
        elif r % 5 == 2:
            u[:] = 1.0                               # the last start of the shortest reader
        inp.u.copy_(torch.from_numpy(u))
        inp.sirs.uniform_(-6, 6)
        inp.snr.uniform_(10, 20)
        pp, st = np.zeros(3, np.int32), np.zeros(3, np.int32)
        for k in range(3):                           # every candidate's first and last start, then the middle
            pp[k], st[k] = probes[k].pop(0) if probes[k] else (r % counts[k + (k > 0)], LEN // 3)
        bad = r == runs - 1
        if bad:                                      # out of range: clamped, and reported alike
            pp[:] = [len(spk) + 3, -2, 99]
            st[:] = [-5, 10 ** 7, 3]
            if dry_picks:
                inp.dry_picks[0, 0] = 7
        inp.probe_pick.copy_(torch.from_numpy(pp))
        inp.probe_start.copy_(torch.from_numpy(st))
        ps.run()
        es = _errors(R)
        pt.run()
        et = _errors(R)
        assert es == et, (r, es, et)
        assert (es is not None) == bad, (r, es)
        _same(os_, ot, r)
    assert not any(probes)
    assert ps.is_graph() and pt.is_graph()


def test_launches_and_side_stream(world):
    render, R = _R()
    spk, noi, mus, pools, dry, gains = world
    inp = Inputs()
    ps, os_ = _plan(render, R, pools["spectra"], inp)
    pt, ot = _plan(render, R, pools["taps"], inp)
    inp.picks.copy_(torch.tensor([[1, 2, 3, 0], [4, 6, 1, 2], [0, 5, 2, 1]], dtype=torch.int32))
    inp.u.uniform_()
    inp.sirs.fill_(2.5)
    inp.snr.fill_(15.0)
    inp.probe_pick.fill_(1)
    inp.probe_start.fill_(777)
    ps.run(); pt.run()                               # graphs captured
    torch.cuda.synchronize()
    n = []
    for p in (ps, pt):
        R.reset_stats()
        p.run()
        n.append(R.launch_count())
    assert n[1] == n[0] + 1, n
    assert ps.is_graph() and pt.is_graph()
    torch.cuda.synchronize()
    ref = {k: [t.clone() for t in v] if isinstance(v, list) else v.clone() for k, v in ot.items()}
    for v in ot.values():
        for t in (v if isinstance(v, list) else [v]):
            t.fill_(-1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(2e7))                  # queued work in front of the run
        pt.run(s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    _same(ref, ot, "side stream")
    _same(os_, ot, "against the spectral host pools")


@pytest.mark.parametrize("case", ["plain", "normalised", "normalised_zero"])
def test_tap_bank_and_whole_stem(case):
    render, R = _R()
    from sonicsim_b200 import _lib
    normalize = case != "plain"
    rng = np.random.default_rng(3 + len(case))
    c = Cand(rng, 50000, 5, 3, 9000)                 # abs-max 0.6: normalised taps are true quotients
    if case == "normalised_zero":
        c.h[:] = 0.0                                 # an all-zero set: stored undivided, rendered as zeros alike
    else:
        assert np.max(np.abs(c.h)) not in (0.0, 1.0)
    K = (c.L + 4095) // 4096
    tb = R.rir_bank(c.h, normalize, TAPS, host=True, form="taps")
    sb = R.rir_bank(c.h, normalize, TAPS, host=True)
    db = R.rir_bank(c.h, normalize, TAPS)
    assert tb.form == "taps" and sb.form == "spectra" and tb.nbytes == 0
    assert tb.host_nbytes == 16384 * c.P * c.C * K + 4 * c.P * c.C
    assert 2 * (tb.host_nbytes - 4 * c.P * c.C) == (sb.host_nbytes - 4 * c.P * c.C) // 2
    want = _lib.SS_BANK_HOST | _lib.SS_BANK_TAPS | _lib.SS_DIRECT_TARGET | (_lib.SS_RIR_NORMALIZE if normalize else 0)
    assert R.lib.ss_bank_flags(tb._h) == want
    ref, ref_d = torch.zeros((3, c.N), device="cuda"), torch.zeros((3, c.N), device="cuda")
    R.render_device([render.MovingSource(to(c.x), db, to(c.b), bounds_host=c.b, direct_taps=TAPS)], [ref],
                    direct_outs=[ref_d])
    for bank in (sb, tb):
        pool = R.source_pool([render.MovingSource(c.x, bank, c.b)])
        pick, y, yd = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros_like(ref), torch.zeros_like(ref)
        plan = R.plan_device([render.Pooled(pool, pick[0], (0, c.N), TAPS)], [y], direct_outs=[yd])
        plan.run()
        torch.cuda.synchronize()
        assert torch.equal(y, ref) and torch.equal(yd, ref_d), bank.form
        assert (case == "normalised_zero") == (not bool(ref.abs().max() > 0))
        plan.close()
        pool.close()


def test_device_memory_of_a_tap_pool():
    render, R = _R()
    rng = np.random.default_rng(11)
    n, P, C, N = 24, 60, 6, 30 * RATE
    b = np.round(np.linspace(0, N, P)).astype(np.int32)
    h = so.synth_rirs(rng, P, C, 4096)
    x = so.synth_dry(rng, N)
    banks = [R.rir_bank(h, host=True, form="taps") for _ in range(n)]
    assert sum(k.host_nbytes for k in banks) == n * 4 * 4096 * P * C
    cands = [render.MovingSource(x, banks[i], b) for i in range(n)]
    R.source_pool(cands, levels="channels").close()   # the context's own render scratch grows to this build's size
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    pool = R.source_pool(cands, levels="channels")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    grown = free0 - torch.cuda.mem_get_info()[0]
    assert pool.nbytes == 40 * n + 4 * n * P + 8 * n, pool.nbytes
    assert grown <= pool.nbytes + (32 << 20), (grown, pool.nbytes)
    assert pool.host_nbytes == n * (4 * N + 8 * (N + 1)), pool.host_nbytes
    pool.close()
    for k in banks:
        k.close()


def test_refusals():
    render, R = _R()
    lib = R.lib
    from sonicsim_b200 import _lib
    rng = np.random.default_rng(5)
    c = Cand(rng, 20000, 3, 2, 4096)
    tb, sb = R.rir_bank(c.h, host=True, form="taps"), R.rir_bank(c.h, host=True)
    with pytest.raises(ValueError, match="needs host=True"):
        R.rir_bank(c.h, form="taps")
    with pytest.raises(ValueError, match="form must be"):
        R.rir_bank(c.h, host=True, form="fp16")
    with pytest.raises(ValueError, match="banks are all of one form"):
        R.source_pool([render.MovingSource(c.x, sb, c.b), render.MovingSource(c.x, tb, c.b)])
    src = render.MovingSource(to(c.x), tb, to(c.b), bounds_host=c.b)
    out = torch.zeros((2, c.N), device="cuda")
    with pytest.raises(ValueError, match="host bank"):
        R.render_device([src], [out])
    with pytest.raises(ValueError, match="host bank"):
        R.plan_device([src], [out])
    # the C ABI
    h = ctypes.c_void_p()
    flags = _lib.SS_BANK_TAPS
    assert lib.ss_bank_create_host(R.ctx, c.h.ctypes.data, c.P, c.C, c.L, flags, 0, ctypes.byref(h)) == \
        _lib.SS_ERR_INVALID and not h.value
    d_h = to(c.h)
    assert lib.ss_bank_create_dev(R.ctx, d_h.data_ptr(), c.P, c.C, c.L, flags | _lib.SS_RIR_NORMALIZE, 0, None,
                                  ctypes.byref(h)) == _lib.SS_ERR_INVALID and not h.value
    item = _lib.SsSource(x=src.dry.data_ptr(), out=out.data_ptr(), bounds=src.bounds.data_ptr(),
                         bounds_host=c.b.ctypes.data, N=c.N, P=c.P, C=2, L=c.L, mode=_lib.SS_MOVING_BOUNDS,
                         rir_bank=tb._h.value)
    assert lib.ss_render_dev(R.ctx, ctypes.byref(item), 1, None) == _lib.SS_ERR_INVALID
    assert lib.ss_plan_create(R.ctx, ctypes.byref(item), 1, ctypes.byref(h)) == _lib.SS_ERR_INVALID and not h.value
    cand = (_lib.SsSource * 2)()
    for i, bank in enumerate((sb, tb)):
        cand[i] = _lib.SsSource(x=src.dry.data_ptr(), bounds_host=c.b.ctypes.data, N=c.N, P=c.P, C=2, L=c.L,
                                mode=_lib.SS_MOVING_BOUNDS, rir_bank=bank._h.value)
    assert lib.ss_pool_create(R.ctx, cand, 2, ctypes.byref(h)) == _lib.SS_ERR_INVALID and not h.value
    cand[0] = cand[1]
    assert lib.ss_pool_create(R.ctx, cand, 2, ctypes.byref(h)) == _lib.SS_OK
    lib.ss_pool_destroy(h)
    tb.close()
    sb.close()
