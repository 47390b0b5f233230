"""Pair gains (Renderer.pair_gains; ss_pair_gains_create, ss_plan_create_pair) through the real kernels.  A pair-gain
table holds the whole-stem loudness gain of every (dry signal, candidate) pair of a pool and a dry pool; a dry-picked
slot with it stores its stems times the picked pair's (float)gain.  Checked:
  1. every pair's (LUFS, gain) equals render_host(..., lufs_targets=[t], loudness_out=) of the pair rendered whole, bit
     for bit, and the float64 BS.1770 oracle within 1e-6 dB; a silent signal (-inf, measured as -40) and unmeasured
     pairs (NaN target: NaN, gain 1) included; the four residencies of pool and dry pool measure the same bits;
  2. over many runs with new picks, dry picks and starts written on the device, every stem and direct stem equals the
     same plan's stem without pair gains times (float)gain, and render_device of the pair at that window times the
     gain, bit for bit: an aligned moving pool with direct sets, a mixed-K pool and a static pool;
  3. host pool and host dry pool forms equal the device forms bit for bit;
  4. on a pool with loudness gains the pair's gain replaces the candidate's; a plain DryPick there is still refused;
  5. clamped picks (bits 3 and 4) take the clamped pair's gain, on k_blocks' and on k_stage's path;
  6. mixtures over pair-gained slots equal ss_mix_dev on the plan's own stems, and start draws give the same starts and
     `used` with and without pair gains;
  7. launches per run equal the same plan without pair gains;
  8. every refusal, in Python and through the C ABI, leaves nothing written;
  9. one plan at the shape of profiles/time_dry_pool.py form (d): 16 examples x (2 speakers + noise), a dry pool of 256
     gappy 60 s streams, pair gains over speakers and noises."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from draw_reference import gappy_dry
from gpu_plumbing import _R, to
from pool_worlds import Cand, DrySlots, _host_pool, _mix_dev, dry_signals, reference
from pool_worlds import world  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

NAN = float("nan")
RATE = 16000


def host_pair(R, render, c, x, t):
    """render_host of candidate c with dry x[:N] and target t: (stem, (LUFS, gain))."""
    xs = x[:c.N].cpu().numpy().copy()
    src = render.MovingSource(xs, c.bank, c.b) if c.b is not None else render.StaticSource(xs, c.bank)
    lo = []
    out = R.render_host([src], lufs_targets=[t], loudness_out=lo, sr=RATE)[0]
    return out, lo[0]


def targets_for(seed, n_dry, n, nan=((1, 0),)):
    t = np.random.default_rng(seed).uniform(-19.0, -15.0, (n_dry, n))
    for d, i in nan:
        t[d, i] = np.nan
    return t


def with_gains(srcs, pg):
    return [s._replace(dry=s.dry._replace(gains=pg)) for s in srcs]


def gain_of(pg, d, i):
    g = pg.loudness[d, i, 1]
    return np.float32(1.0) if np.isnan(g) else np.float32(g)


def test_pair_loudness_equals_render_host_and_the_oracle(world):
    render, R = _R()
    cands, _ = world["speakers"]
    n_max = max(c.N for c in cands)
    sig = dry_signals(601, 3, n_max, 0)
    sig[2].zero_()                                            # silent: -inf LUFS, measured as -40
    t = targets_for(602, 3, len(cands), nan=((1, 0), (0, 3)))
    pools = {"device": R.source_pool([c.src for c in cands]), "host": _host_pool(R, render, cands, 40)}
    dpools = {"device": R.dry_pool(sig), "host": R.dry_pool([s.cpu().numpy() for s in sig], host=True)}
    tabs = []
    try:
        for pr in ("device", "host"):
            for dr_ in ("device", "host"):
                tabs.append(R.pair_gains(pools[pr], dpools[dr_], t, sr=RATE))
        L = tabs[0].loudness
        assert L.shape == (3, len(cands), 2) and L.dtype == np.float64 and tabs[0].nbytes == 4 * 3 * len(cands)
        for g in tabs[1:]:                                    # every residency measures the same bits
            assert np.array_equal(g.loudness, L, equal_nan=True)
        for d in range(3):
            for i, c in enumerate(cands):
                if np.isnan(t[d, i]):
                    assert np.isnan(L[d, i]).all()
                    continue
                _, lo = host_pair(R, render, c, sig[d], t[d, i])
                assert (L[d, i, 0], L[d, i, 1]) == tuple(lo), (d, i, L[d, i], lo)            # -inf == -inf
                if d == 2:
                    assert np.isneginf(L[d, i, 0])
                    assert L[d, i, 1] == pytest.approx(10.0 ** ((t[d, i] + 40.0) / 20.0), rel=1e-15)
                    continue
                stem, _ = reference(c, sig[d], 0, c.N, 0)
                ref = so.bs1770_integrated_loudness(stem.cpu().numpy().T.astype(np.float64), RATE, 0.4,
                                                    up_to_8_channels=True)
                assert abs(L[d, i, 0] - ref) < 1e-6, (d, i, L[d, i, 0], ref)
    finally:
        for g in tabs:
            g.close()
        for p in list(pools.values()) + list(dpools.values()):
            p.close()


def run_pair(plan_g, sl_g, plan_p, sl_p, gen, n, n_dry, n_min, runs, fix=None):
    """Runs both plans (the second without pair gains) on the same picks and starts; returns their snapshots."""
    out = []
    for run in range(runs):
        sl_g.fill(gen, n, n_dry, n_min)
        if fix is not None and run == 0:
            fix(sl_g)
        for a, b in ((sl_p.picks, sl_g.picks), (sl_p.dpicks, sl_g.dpicks), (sl_p.starts, sl_g.starts)):
            a.copy_(b)
        for o in sl_p.outs + (sl_p.douts or []):
            o.fill_(NAN)
        plan_g.run()
        plan_p.run()
        out.append((sl_g.snap(), sl_p.snap()))
    return out


def check_scaled(R, pg, sl, snaps, signals, what, refs=True):
    for r, (sg, sp) in enumerate(snaps):
        for j in range(sl.k):
            i, d, s = int(sg["picks"][j]), int(sg["dpicks"][j]), int(sg["starts"][j])
            g = torch.tensor(gain_of(pg, d, i), device="cuda")
            pairs = [(sg["outs"][j], sp["outs"][j])] + ([(sg["douts"][j], sp["douts"][j])] if sl.taps else [])
            for y, y0 in pairs:
                assert torch.isfinite(y).all(), (what, r, j)
                assert torch.equal(y, y0 * g), (what, r, j, i, d, s)
            if refs:
                ref, dref = reference(sl.cands[i], signals[d], s, sl.wl, sl.taps)
                assert torch.equal(sg["outs"][j], ref * g), (what, r, j)
                if sl.taps:
                    assert torch.equal(sg["douts"][j], dref * g), (what, r, j)


@pytest.mark.parametrize("kind", ["speakers", "long", "noise"])
def test_stems_are_the_plain_stems_times_the_pair_gain(world, kind):
    render, R = _R()
    cands, taps = world[kind]
    n_max = max(c.N for c in cands)
    signals = dry_signals(611, 5, n_max, 3001)
    pool, dpool = R.source_pool([c.src for c in cands]), R.dry_pool(signals)
    pg = R.pair_gains(pool, dpool, targets_for(612, 5, len(cands)), sr=RATE)
    wl = 9000 if kind != "noise" else 20000
    sl_g, sl_p = DrySlots(pool, dpool, cands, wl, taps), DrySlots(pool, dpool, cands, wl, taps)
    plan_g = R.plan_device(with_gains(sl_g.srcs, pg), sl_g.outs, direct_outs=sl_g.douts)
    plan_p = R.plan_device(sl_p.srcs, sl_p.outs, direct_outs=sl_p.douts)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(613)

    def fix(sl):                                              # the unmeasured pair (1, 0): gain 1
        sl.picks[0] = 0
        sl.dpicks[0] = 1
    try:
        snaps = run_pair(plan_g, sl_g, plan_p, sl_p, gen, len(cands), dpool.n, min(c.N for c in cands), 8, fix)
        assert plan_g.is_graph()
        torch.cuda.synchronize()
        R.check_device_errors()
        check_scaled(R, pg, sl_g, snaps, signals, kind)
        picked = {(int(p), int(d)) for sg, _ in snaps for p, d in zip(sg["picks"], sg["dpicks"])}
        assert len(picked) >= 12, picked
        # launches per run equal the same plan without pair gains
        counts = []
        for p in (plan_g, plan_p):
            torch.cuda.synchronize()
            R.reset_stats()
            p.run()
            torch.cuda.synchronize()
            counts.append(R.launch_count())
        assert counts[0] == counts[1], counts
    finally:
        for o in (plan_g, plan_p, pg, pool, dpool):
            o.close()


def test_host_forms_equal_the_device_form(world):
    render, R = _R()
    cands, taps = world["speakers"]
    n_max = max(c.N for c in cands)
    sig = dry_signals(621, 4, n_max, 0)
    t = targets_for(622, 4, len(cands))
    pools = {"device": R.source_pool([c.src for c in cands]), "host": _host_pool(R, render, cands, taps)}
    dpools = {"device": R.dry_pool(sig), "host": R.dry_pool([s.cpu().numpy() for s in sig], host=True)}
    wl = 9000
    forms, held = {}, []
    try:
        for pr, dr_ in (("device", "device"), ("device", "host"), ("host", "host")):
            pg = R.pair_gains(pools[pr], dpools[dr_], t, sr=RATE)
            sl = DrySlots(pools[pr], dpools[dr_], cands, wl, taps)
            plan = R.plan_device(with_gains(sl.srcs, pg), sl.outs, direct_outs=sl.douts)
            held += [plan, pg]
            forms[(pr, dr_)] = (sl, plan)
        base, plan0 = forms[("device", "device")]
        gen = torch.Generator(device="cuda")
        gen.manual_seed(623)
        for run in range(5):
            base.fill(gen, len(cands), 4, min(c.N for c in cands))
            if run == 1:                                      # clamped picks on every path: bits 3 and 4
                base.picks.copy_(torch.tensor([-1, len(cands), 1, 99], dtype=torch.int32))
                base.dpicks.copy_(torch.tensor([7, -3, 1 << 30, 0], dtype=torch.int32))
            plan0.run()
            want = base.snap()
            for key, (sl, plan) in forms.items():
                if sl is base:
                    continue
                for a, b in ((sl.picks, base.picks), (sl.dpicks, base.dpicks), (sl.starts, base.starts)):
                    a.copy_(b)
                for o in sl.outs + sl.douts:
                    o.fill_(NAN)
                plan.run()
                got = sl.snap()
                for a, b in zip(got["outs"] + got["douts"], want["outs"] + want["douts"]):
                    assert torch.equal(a, b), (key, run)
            if run == 1:
                torch.cuda.synchronize()
                with pytest.raises(IndexError):
                    R.check_device_errors()
                n, n_dry = len(cands), 4
                cl = [(min(max(p, 0), n - 1), min(max(d, 0), n_dry - 1))
                      for p, d in zip(want["picks"].tolist(), want["dpicks"].tolist())]
                pg0 = held[1]
                for j, (i, d) in enumerate(cl):
                    ref, dref = reference(cands[i], sig[d], int(want["starts"][j]), wl, taps)
                    g = torch.tensor(gain_of(pg0, d, i), device="cuda")
                    assert torch.equal(want["outs"][j], ref * g) and torch.equal(want["douts"][j], dref * g), j
        torch.cuda.synchronize()
        R.check_device_errors()
    finally:
        for o in held + list(pools.values()) + list(dpools.values()):
            o.close()


def test_pair_gain_replaces_the_pool_gain(world):
    render, R = _R()
    cands, taps = world["speakers"]
    n_max = max(c.N for c in cands)
    sig = dry_signals(631, 3, n_max, 0)
    t = targets_for(632, 3, len(cands))
    plain = R.source_pool([c.src for c in cands])
    gpool = R.source_pool([c.src for c in cands], lufs_targets=[-30.0] * len(cands), sr=RATE)
    dpool = R.dry_pool(sig)
    pg_plain, pg_gain = R.pair_gains(plain, dpool, t, sr=RATE), R.pair_gains(gpool, dpool, t, sr=RATE)
    assert np.array_equal(pg_plain.loudness, pg_gain.loudness, equal_nan=True)
    sl_a, sl_b = DrySlots(gpool, dpool, cands, 9000, taps), DrySlots(plain, dpool, cands, 9000, taps)
    held = [pg_plain, pg_gain, plain, gpool, dpool]
    try:
        with pytest.raises(ValueError, match="loudness gains"):
            R.plan_device(sl_a.srcs, sl_a.outs, direct_outs=sl_a.douts)
        # the C ABI refuses a plain dry pick on a gains pool, and takes it with pair gains
        items, n, keep = R._device_items(sl_a.srcs, sl_a.outs, sl_a.douts)
        arr = R._device_dry(with_gains(sl_a.srcs, pg_gain))
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_dry(R.ctx, items, n, None, 0, None, 0, arr, len(arr), ctypes.byref(h)) == \
            -1 and not h.value
        tabs = (ctypes.c_void_p * len(arr))(*[pg_gain._h.value] * len(arr))
        assert R.lib.ss_plan_create_pair(R.ctx, items, n, None, 0, None, 0, arr, tabs, len(arr), ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)
        plan_a = R.plan_device(with_gains(sl_a.srcs, pg_gain), sl_a.outs, direct_outs=sl_a.douts)
        plan_b = R.plan_device(with_gains(sl_b.srcs, pg_plain), sl_b.outs, direct_outs=sl_b.douts)
        held = [plan_a, plan_b] + held
        gen = torch.Generator(device="cuda")
        gen.manual_seed(633)
        snaps = run_pair(plan_a, sl_a, plan_b, sl_b, gen, len(cands), 3, min(c.N for c in cands), 4)
        torch.cuda.synchronize()
        for sa, sb in snaps:                                  # the pool's gains play no part
            for a, b in zip(sa["outs"] + sa["douts"], sb["outs"] + sb["douts"]):
                assert torch.equal(a, b)
        sa = snaps[-1][0]
        for j in range(sl_a.k):
            i, d, s = int(sa["picks"][j]), int(sa["dpicks"][j]), int(sa["starts"][j])
            ref, dref = reference(cands[i], sig[d], s, 9000, taps)
            g = torch.tensor(gain_of(pg_gain, d, i), device="cuda")
            assert torch.equal(sa["outs"][j], ref * g) and torch.equal(sa["douts"][j], dref * g), j
        R.check_device_errors()
    finally:
        for o in held:
            o.close()


def test_mixtures_and_draws_over_pair_gained_slots(world):
    render, R = _R()
    spk, _ = world["speakers"]
    noi, _ = world["noise"]
    n_max = max(c.N for c in spk + noi)
    rng = np.random.default_rng(641)
    signals = [to(gappy_dry(rng, n_max + 5000)) for _ in range(6)]
    sp, npool = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])
    dpool = R.dry_pool(signals, levels=True)
    pg_s = R.pair_gains(sp, dpool, targets_for(642, 6, len(spk)), sr=RATE)
    pg_n = R.pair_gains(npool, dpool, targets_for(643, 6, len(noi), nan=()) - 7.0, sr=RATE)
    wl, B, TR = 12000, 4, 101
    picks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    sirs, snr = torch.zeros((B, 1), device="cuda"), torch.zeros(B, device="cuda")
    u = torch.zeros((B, TR), dtype=torch.float64, device="cuda")

    def build(gains):
        starts = torch.zeros(B, dtype=torch.int32, device="cuda")
        used = torch.zeros(B, dtype=torch.int32, device="cuda")
        outs = [torch.empty((2, wl), device="cuda") for _ in range(3 * B)]
        mix, spo = torch.empty((B, 2, wl), device="cuda"), torch.empty((B, 2, 2, wl), device="cuda")
        srcs, mixes, draws = [], [], []
        for b in range(B):
            for j, (pl, pg) in enumerate(((sp, pg_s), (sp, pg_s), (npool, pg_n))):
                srcs.append(render.Pooled(pl, picks[b, j], (starts[b], wl), 0,
                                          render.DryPick(dpool, dpicks[b, j], pg if gains else None)))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sirs[b], snr[b], mix[b], spo[b]))
            draws.append(render.CropDraw(starts[b], [3 * b, 3 * b + 1], u[b], used[b]))
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), outs, mix, spo, starts, used

    plan_g, outs_g, mix_g, spo_g, st_g, used_g = build(True)
    plan_p, outs_p, _, _, st_p, used_p = build(False)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(644)
    try:
        counts = []
        for run in range(4):
            picks[:, :2].copy_(torch.randint(0, len(spk), (B, 2), generator=gen, device="cuda", dtype=torch.int32))
            picks[:, 2].copy_(torch.randint(0, len(noi), (B,), generator=gen, device="cuda", dtype=torch.int32))
            dpicks.copy_(torch.randint(0, dpool.n, (B, 3), generator=gen, device="cuda", dtype=torch.int32))
            u.uniform_(generator=gen)
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(10, 20, generator=gen)
            torch.cuda.synchronize()
            R.reset_stats()
            plan_g.run()
            torch.cuda.synchronize()
            counts.append(R.launch_count())
            R.reset_stats()
            plan_p.run()
            torch.cuda.synchronize()
            counts.append(R.launch_count())
            assert torch.equal(st_g, st_p) and torch.equal(used_g, used_p), run
            for b in range(B):
                for j, pg in enumerate((pg_s, pg_s, pg_n)):
                    g = torch.tensor(gain_of(pg, int(dpicks[b, j]), int(picks[b, j])), device="cuda")
                    assert torch.equal(outs_g[3 * b + j], outs_p[3 * b + j] * g), (run, b, j)
                m, s = _mix_dev(R, torch.stack([outs_g[3 * b].reshape(-1), outs_g[3 * b + 1].reshape(-1)]),
                                outs_g[3 * b + 2].reshape(1, -1), sirs[b], snr[b])
                assert torch.equal(mix_g[b].reshape(-1), m), (run, b)
                assert torch.equal(spo_g[b].reshape(2, -1), s), (run, b)
        assert len(set(counts[1:])) == 1, counts                # the first run captures the graphs
        assert int(used_p.min()) >= 0
        R.check_device_errors()
    finally:
        for o in (plan_g, plan_p, pg_s, pg_n, sp, npool, dpool):
            o.close()


def test_refusals_write_nothing(world):
    render, R = _R()
    from sonicsim_b200 import _lib as L
    cands, _ = world["long"]
    n_max = max(c.N for c in cands)
    sig = dry_signals(651, 2, n_max, 0)
    pool, dpool, short = R.source_pool([c.src for c in cands]), R.dry_pool(sig), R.dry_pool([sig[0][:n_max - 1]])
    other = R.source_pool([c.src for c in cands[:2]])
    held = [pool, dpool, short, other]
    try:
        # Python: checked before any C call
        with pytest.raises(ValueError, match="shorter than the pool's longest"):
            R.pair_gains(pool, short, -20.0)
        with pytest.raises(ValueError, match="not finite"):
            R.pair_gains(pool, dpool, np.full((2, len(cands)), np.inf))
        with pytest.raises(ValueError, match="\\(n_dry, n\\)"):
            R.pair_gains(pool, dpool, np.zeros((len(cands), 2)))
        pg = R.pair_gains(pool, dpool, -20.0, sr=RATE)
        held.insert(0, pg)
        # a PairGains of another pool, or of another dry pool, in a plan
        sl = DrySlots(other, dpool, cands[:2], 3000, 0, k=2)
        with pytest.raises(ValueError, match="another SourcePool or DryPool"):
            R.plan_device(with_gains(sl.srcs, pg), sl.outs)
        pg.close()
        with pytest.raises(ValueError, match="is closed"):
            R.plan_device(with_gains(DrySlots(pool, dpool, cands, 3000, 0, k=2).srcs, pg), sl.outs)
        pg = R.pair_gains(pool, dpool, -20.0, sr=RATE)
        held.insert(0, pg)

        # the C ABI: every refusal leaves results and *out untouched
        n, n_dry = len(cands), 2
        from sonicsim_b200.SonicSim_audio import gating_block_size, gating_plan
        plans = {}
        post = (L.SsPostLufs * n)()
        for i, c in enumerate(cands):
            bs = float(gating_block_size(c.N, RATE))
            plans[i] = gating_plan(c.N, float(RATE), bs)
            brk, blo, bhi = plans[i]
            post[i] = L.SsPostLufs(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data,
                                   n_e=len(brk) - 1, n_blocks=len(blo), rate=float(RATE), block_size=bs)
        t = np.full((n_dry, n), -20.0)

        def c_call(p=pool._h, d=dpool._h, ps=post, tg=None, want=L.SS_ERR_INVALID):
            res = np.full((n_dry, n, 2), 1234.5)
            h = ctypes.c_void_p()
            tg = t if tg is None else tg
            got = R.lib.ss_pair_gains_create(R.ctx, p, d, ps, tg.ctypes.data, res.ctypes.data, ctypes.byref(h))
            assert got == want and not h.value and (res == 1234.5).all(), got
        c_call(p=None)
        c_call(d=None)
        c_call(ps=None)
        c_call(d=short._h)
        bad = np.array(t)
        bad[1, 2] = -np.inf
        c_call(tg=bad)
        for field, v in (("n_e", 0), ("rate", 0.0), ("block_size", NAN), ("blk_lo", None)):
            ps = (L.SsPostLufs * n)(*post)
            setattr(ps[1], field, v)
            c_call(ps=ps)
        # more than 2^26 pairs: a dry pool of 2^24 copies of one signal over 5 candidates (refused before any target
        # is read)
        big_n = 1 << 24
        ptrs = np.full(big_n, sig[0].data_ptr(), np.uint64)
        lens = np.full(big_n, sig[0].numel(), np.int32)
        hb = ctypes.c_void_p()
        assert R.lib.ss_dry_pool_create(R.ctx, ptrs.ctypes.data, lens.ctypes.data, big_n, 0, ctypes.byref(hb)) == 0
        five = R.source_pool([c.src for c in cands] + [cands[0].src])
        held.append(five)
        try:
            c_call(p=five._h, d=hb, ps=(L.SsPostLufs * 5)(*post, post[0]), want=L.SS_ERR_UNSUPPORTED)
        finally:
            R.lib.ss_dry_pool_destroy(hb)
        # C > 8
        rng = np.random.default_rng(652)
        wide = Cand(so.synth_dry(rng, 9000), so.synth_rirs(rng, 1, 9, 300)[0], None)
        wpool = R.source_pool([wide.src])
        held.append(wpool)
        c_call(p=wpool._h, ps=(L.SsPostLufs * 1)(post[0]), tg=np.full(2, -20.0), want=L.SS_ERR_UNSUPPORTED)
        # plans: a table of another pool or another dry pool than the pick's
        sl = DrySlots(pool, dpool, cands, 3000, 0, k=2)
        items, ni, keep = R._device_items(sl.srcs, sl.outs)
        arr = R._device_dry(sl.srcs)
        pg_other = R.pair_gains(other, dpool, -20.0, sr=RATE)
        dpool2 = R.dry_pool(sig)
        pg_dry2 = R.pair_gains(pool, dpool2, -20.0, sr=RATE)
        held = [pg_other, pg_dry2, dpool2] + held
        for bad_tab in (pg_other, pg_dry2):
            tabs = (ctypes.c_void_p * 2)(pg._h.value, bad_tab._h.value)
            h = ctypes.c_void_p()
            assert R.lib.ss_plan_create_pair(R.ctx, items, ni, None, 0, None, 0, arr, tabs, 2, ctypes.byref(h)) == \
                L.SS_ERR_INVALID and not h.value
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_pair(R.ctx, items, ni, None, 0, None, 0, arr, None, 2, ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)
    finally:
        for o in held:
            o.close()


def test_training_scale_plan_of_form_d():
    """16 examples x (2 dry-picked speakers + a dry-picked noise) over a dry pool of 256 gappy 60 s streams, with draws
    and mixtures, pair gains over speakers and noises: every stem equals the same plan's stem without pair gains times
    the pair's gain, starts and `used` are the same, and a sample of pairs meets render_host's loudness bit for bit."""
    render, R = _R()
    rng = np.random.default_rng(661)
    U, S, CROP, N_DRY, TR = 16, 2, 4 * RATE, 256, 101
    spk = []
    for j in range(8):
        P, N = 3 + j % 3, 30 * RATE + 997 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        spk.append(Cand(gappy_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    noi = [Cand(so.synth_dry(rng, 30 * RATE + 503 * j) * np.float32(0.3), so.synth_rirs(rng, 1, 2, 4096)[0], None)
           for j in range(4)]
    signals = [to(gappy_dry(rng, 60 * RATE)) for _ in range(N_DRY)]
    torch.cuda.synchronize()
    sp, npool = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])
    dpool = R.dry_pool(signals, levels=True)
    t_s = rng.uniform(-19, -15, (N_DRY, len(spk)))
    t_n = rng.uniform(-26, -22, (N_DRY, len(noi)))
    pg_s, pg_n = R.pair_gains(sp, dpool, t_s, sr=RATE), R.pair_gains(npool, dpool, t_n, sr=RATE)
    picks = torch.zeros((U, S + 1), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((U, S + 1), dtype=torch.int32, device="cuda")
    sirs, snr = torch.zeros((U, S - 1), device="cuda"), torch.zeros(U, device="cuda")
    u = torch.zeros((U, TR), dtype=torch.float64, device="cuda")

    def build(gains):
        starts = torch.zeros(U, dtype=torch.int32, device="cuda")
        used = torch.zeros(U, dtype=torch.int32, device="cuda")
        outs = [torch.empty((2, CROP), device="cuda") for _ in range(U * (S + 1))]
        mix, spo = torch.empty((U, CROP), device="cuda"), torch.empty((U, S, CROP), device="cuda")
        srcs, mixes, draws = [], [], []
        for e in range(U):
            for k, (pl, pg) in enumerate(((sp, pg_s), (sp, pg_s), (npool, pg_n))):
                srcs.append(render.Pooled(pl, picks[e, k], (starts[e], CROP), 0,
                                          render.DryPick(dpool, dpicks[e, k], pg if gains else None)))
            base = (S + 1) * e
            mixes.append(render.Mixture([base, base + 1], [base + 2], sirs[e], snr[e], mix[e], spo[e], mono=True))
            draws.append(render.CropDraw(starts[e], [base, base + 1], u[e], used[e]))
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), outs, mix, starts, used

    plan_g, outs_g, mix_g, st_g, used_g = build(True)
    plan_p, outs_p, mix_p, st_p, used_p = build(False)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(662)
    try:
        for step in range(6):
            sc = torch.randint(0, len(spk) // 2, (U,), generator=gen, device="cuda", dtype=torch.int32)
            picks[:, :S].copy_(2 * sc[:, None] + torch.rand(U, S, generator=gen, device="cuda").argsort(1).int())
            picks[:, S].copy_(torch.randint(0, len(noi), (U,), generator=gen, device="cuda", dtype=torch.int32))
            dpicks.copy_(torch.randint(0, N_DRY, (U, S + 1), generator=gen, device="cuda", dtype=torch.int32))
            u.uniform_(generator=gen)
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(10, 20, generator=gen)
            plan_g.run()
            plan_p.run()
            torch.cuda.synchronize()
            assert torch.equal(st_g, st_p) and torch.equal(used_g, used_p), step
            for e in range(U):
                for k, pg in enumerate((pg_s, pg_s, pg_n)):
                    g = torch.tensor(gain_of(pg, int(dpicks[e, k]), int(picks[e, k])), device="cuda")
                    y = outs_g[(S + 1) * e + k]
                    assert torch.isfinite(y).all() and torch.equal(y, outs_p[(S + 1) * e + k] * g), (step, e, k)
        R.check_device_errors()
        Ls, Ln = pg_s.loudness, pg_n.loudness
        assert np.isfinite(Ls).all() and np.isfinite(Ln).all()
        for d, i in ((0, 0), (N_DRY - 1, len(spk) - 1), (128, 3)):
            _, lo = host_pair(R, render, spk[i], signals[d], t_s[d, i])
            assert (Ls[d, i, 0], Ls[d, i, 1]) == tuple(lo), (d, i)
        _, lo = host_pair(R, render, noi[2], signals[77], t_n[77, 2])
        assert (Ln[77, 2, 0], Ln[77, 2, 1]) == tuple(lo)
        assert pg_s.nbytes == 4 * N_DRY * len(spk) and pg_n.nbytes == 4 * N_DRY * len(noi)
    finally:
        for o in (plan_g, plan_p, pg_s, pg_n, sp, npool, dpool):
            o.close()
