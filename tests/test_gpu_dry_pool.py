"""Dry pools (Renderer.dry_pool; ss_dry_pool) and dry-picked pooled slots (render.DryPick; ss_plan_create_dry) through
the real kernels.  A dry-picked slot renders, at every run, its pool's picked candidate with the dry signal its own dry
pick names.  Checked:
  1. bits: an aligned moving pool with direct stems, a pool whose candidates differ in K, and a static pool, over dry
     signals longer than the longest candidate whose tails are NaN; many runs with new picks, dry picks and starts written
     on the device and no host synchronisation in between; every stem and direct stem equals render_device of the picked
     candidate with dry = signal[:N] at the same fixed window, bit for bit, and is finite;
  2. mixtures over dry-picked slots equal ss_mix_dev on the plan's own stems;
  3. draws over gappy dry signals (create_long_audio's layout): every start and `used` equals tests/draw_reference.py on
     the device's dry tables, with dry-picked and pooled speakers in one draw; the dry tables equal a long-double prefix
     sum within the bound of test_gpu_plan_draw.py;
  4. a dry pick out of range sets bit 4 (IndexError) and renders the clamped signal;
  5. launches per run equal with and without dry picks; the no-graph and profiling paths give the same bits; a side
     stream behind queued work;
  6. every refusal, in Python and through the C ABI, with nothing written;
  7. one plan at the shape of profiles/time_draw_step.py: 16 examples x (2 speakers + noise), 256 dry streams of 60 s."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
import draw_reference as dr
from draw_reference import NEAR_DB, TABLE_TOL
from gpu_plumbing import _R, to
from pool_worlds import Cand, DrawStep, DrySlots, _mix_dev, dry_signals, reference
from pool_worlds import draw_world, world  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

TAPS = 40
NAN = float("nan")
RATE = 16000
SLEEP = int(5e8)


@pytest.mark.parametrize("kind", ["speakers", "long", "noise"])
def test_bits_equal_render_device(world, kind):
    render, R = _R()
    cands, taps = world[kind]
    n_max = max(c.N for c in cands)
    signals = dry_signals(311, 5, n_max, 3001)
    pool = R.source_pool([c.src for c in cands])
    dpool = R.dry_pool(signals)
    assert dpool.n == 5 and dpool.n_min == n_max + 3001 and not dpool.levels and dpool.nbytes == 8 * 5
    wl = 9000 if kind != "noise" else 20000
    sl = DrySlots(pool, dpool, cands, wl, taps)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(17)
    n_min = min(c.N for c in cands)
    try:
        snaps = []
        for run in range(8):
            sl.fill(gen, len(cands), dpool.n, n_min)
            plan.run()
            snaps.append(sl.snap())
        assert plan.is_graph()
        torch.cuda.synchronize()
        R.check_device_errors()
        for r, snap in enumerate(snaps):
            sl.check(snap, signals, "%s run %d" % (kind, r))
        picked = {(int(p), int(d)) for sn in snaps for p, d in zip(sn["picks"], sn["dpicks"])}
        assert len(picked) >= 12, picked                    # many (trajectory, dry signal) pairs
    finally:
        plan.close()
        pool.close()
        dpool.close()


def test_mixtures_over_dry_picked_slots(world):
    render, R = _R()
    spk, _ = world["speakers"]
    noi, _ = world["noise"]
    n_max = max(c.N for c in spk + noi)
    signals = dry_signals(312, 4, n_max, 100)
    sp, npool, dpool = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi]), R.dry_pool(signals)
    wl, B = 12000, 3
    picks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    starts = torch.zeros(B, dtype=torch.int32, device="cuda")
    sirs = torch.zeros((B, 1), device="cuda")
    snr = torch.zeros(B, device="cuda")
    outs = [torch.empty((2, wl), device="cuda") for _ in range(3 * B)]
    mix = torch.empty((B, 2, wl), device="cuda")
    spo = torch.empty((B, 2, 2, wl), device="cuda")
    srcs, mixtures = [], []
    for b in range(B):
        for j, pl in enumerate((sp, sp, npool)):
            srcs.append(render.Pooled(pl, picks[b, j], (starts[b], wl), 0, render.DryPick(dpool, dpicks[b, j])))
        mixtures.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sirs[b], snr[b], mix[b], spo[b]))
    plan = R.plan_device(srcs, outs, mixtures=mixtures)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(18)
    n_min = min(c.N for c in spk + noi)
    try:
        for run in range(3):
            picks[:, :2].copy_(torch.randint(0, len(spk), (B, 2), generator=gen, device="cuda", dtype=torch.int32))
            picks[:, 2].copy_(torch.randint(0, len(noi), (B,), generator=gen, device="cuda", dtype=torch.int32))
            dpicks.copy_(torch.randint(0, dpool.n, (B, 3), generator=gen, device="cuda", dtype=torch.int32))
            starts.copy_(torch.randint(0, n_min - wl + 1, (B,), generator=gen, device="cuda", dtype=torch.int32))
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(10, 20, generator=gen)
            plan.run()
            torch.cuda.synchronize()
            for b in range(B):
                for j, cs in enumerate((spk, spk, noi)):
                    c = cs[int(picks[b, j])]
                    ref, _ = reference(c, signals[int(dpicks[b, j])], int(starts[b]), wl, 0)
                    assert torch.equal(outs[3 * b + j], ref), (run, b, j)
                m, s = _mix_dev(R, torch.stack([outs[3 * b].reshape(-1), outs[3 * b + 1].reshape(-1)]),
                                outs[3 * b + 2].reshape(1, -1), sirs[b], snr[b])
                assert torch.equal(mix[b].reshape(-1), m), (run, b)
                assert torch.equal(spo[b].reshape(2, -1), s), (run, b)
        R.check_device_errors()
    finally:
        plan.close()
        for p in (sp, npool, dpool):
            p.close()


LEN = 4 * RATE


@pytest.fixture(scope="module")
def draw_pools(draw_world):
    _, R = _R()
    spk, noi, dry = draw_world
    sp = R.source_pool([c.src for c in spk], levels="mono")
    npool = R.source_pool([c.src for c in noi])
    dry_dev = [to(x) for x in dry]
    dpool = R.dry_pool(dry_dev, levels=True)
    Tp = [sp.level_table(i).cpu().numpy() for i in range(sp.n)]
    Td = [dpool.level_table(i).cpu().numpy() for i in range(dpool.n)]
    yield sp, npool, dpool, dry_dev, Tp, Td
    for p in (sp, npool, dpool):
        p.close()


def test_dry_tables(draw_world, draw_pools):
    _, R = _R()
    _, _, dry = draw_world
    sp, npool, dpool, dry_dev, Tp, Td = draw_pools
    assert dpool.levels and dpool.nbytes == 8 * dpool.n + 8 * sum(len(x) + 1 for x in dry) + 8 * dpool.n
    again = R.dry_pool(dry_dev, levels=True)
    try:
        for i, x in enumerate(dry):
            assert torch.equal(again.level_table(i), dpool.level_table(i)), i
            ref = dr.level_table(x[None], True, np.longdouble)
            q = Td[i]
            assert q.shape == (len(x) + 1,) and q[0] == 0.0
            err = float(np.max(np.abs(q.astype(np.longdouble) - ref)))
            assert err <= TABLE_TOL * float(ref[-1]), (i, err / float(ref[-1]))
    finally:
        again.close()
    plain = R.dry_pool(dry_dev)
    assert not plain.levels and plain.level_table(0) is None and plain.nbytes == 8 * plain.n
    plain.close()


@pytest.mark.parametrize("mixed", [True, False])
def test_draws_equal_the_reference(draw_world, draw_pools, mixed):
    render, R = _R()
    spk, noi, _ = draw_world
    sp, npool, dpool, dry_dev, Tp, Td = draw_pools
    st = DrawStep(R, render, sp, npool, dpool, B=12, mixed=mixed)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(19 + mixed)
    try:
        snaps = []
        for run in range(8):
            st.fill(gen, len(spk), len(noi), dpool.n)
            st.plan.run()
            snaps.append(st.snap())
        torch.cuda.synchronize()
        R.check_device_errors()
        total = near = 0
        outcomes = set()
        for r, snap in enumerate(snaps):
            c, n = st.check(snap, spk, noi, dry_dev, Tp, Td, "run %d" % r)
            total, near = total + c, near + n
            outcomes |= {"first" if v == 1 else "later" if v > 1 else "none" for v in snap["used"].cpu().numpy()}
        assert near <= 0.05 * (total + near), (near, total)
        assert total >= 80
        assert {"first", "later"} <= outcomes, outcomes
    finally:
        st.plan.close()


def test_all_silent_takes_the_last_try(draw_world, draw_pools):
    render, R = _R()
    spk, noi, _ = draw_world
    sp, npool, dpool, dry_dev, Tp, Td = draw_pools
    st = DrawStep(R, render, sp, npool, dpool, B=4, mixed=False, thr=100.0, tries=37)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(23)
    try:
        st.fill(gen, len(spk), len(noi), dpool.n)
        st.plan.run()
        snap = st.snap()
        torch.cuda.synchronize()
        assert (snap["used"] == 0).all()
        st.check(snap, spk, noi, dry_dev, Tp, Td, "silent")
    finally:
        st.plan.close()


def test_clamped_dry_pick(world):
    render, R = _R()
    cands, taps = world["speakers"]
    signals = dry_signals(313, 3, max(c.N for c in cands), 7)
    pool, dpool = R.source_pool([c.src for c in cands]), R.dry_pool(signals)
    sl = DrySlots(pool, dpool, cands, 5000, taps, k=2)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    try:
        torch.cuda.synchronize()
        R.check_device_errors()
        for bad, want in ((3, 2), (-5, 0), (1 << 30, 2)):
            sl.picks.copy_(torch.tensor([1, 2], dtype=torch.int32))
            sl.dpicks.copy_(torch.tensor([bad, 1], dtype=torch.int32))
            sl.starts.copy_(torch.tensor([77, 0], dtype=torch.int32))
            plan.run()
            torch.cuda.synchronize()
            with pytest.raises(IndexError, match="dry pick"):
                R.check_device_errors()
            R.check_device_errors()                          # cleared
            snap = sl.snap()
            snap["dpicks"][0] = want
            sl.check(snap, signals, "clamped %d" % bad)
    finally:
        plan.close()
        pool.close()
        dpool.close()


def _bits(sl):
    return [o.clone() for o in sl.outs + (sl.douts or [])]


def test_launches_paths_and_side_stream(world):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    cands, taps = world["speakers"]
    signals = dry_signals(314, 4, max(c.N for c in cands), 50)
    pool, dpool = R.source_pool([c.src for c in cands]), R.dry_pool(signals)
    sl = DrySlots(pool, dpool, cands, 7000, taps)
    bare_sl = DrySlots(pool, dpool, cands, 7000, taps, dry=False)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    bare = R.plan_device(bare_sl.srcs, bare_sl.outs, direct_outs=bare_sl.douts)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(29)
    n_min = min(c.N for c in cands)
    try:
        sl.fill(gen, len(cands), dpool.n, n_min)
        plan.run()
        ref = _bits(sl)
        c0 = R.launch_count()
        plan.run()
        with_dry = R.launch_count() - c0
        bare.run()
        c0 = R.launch_count()
        bare.run()
        assert with_dry == R.launch_count() - c0 and plan.is_graph() and bare.is_graph()
        for a, b in zip(ref, _bits(sl)):
            assert torch.equal(a, b)
        # profiling: the same bits
        for o in sl.outs + sl.douts:
            o.fill_(NAN)
        R.set_profiling(True)
        try:
            plan.run()
            R.get_profile()
        finally:
            R.set_profiling(False)
        for a, b in zip(ref, _bits(sl)):
            assert torch.equal(a, b)
        snap = sl.snap()
        torch.cuda.synchronize()
        sl.check(snap, signals, "profiling")
        # a side stream behind queued work, with the picks written on it
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            for o in sl.outs + sl.douts:
                o.fill_(NAN)
            sl.dpicks.fill_(0)
            torch.cuda._sleep(SLEEP)
            sl.fill(gen, len(cands), dpool.n, n_min)
            plan.run(stream=s.cuda_stream)
            busy = not s.query()
            snap = sl.snap()
        assert busy
        s.synchronize()
        sl.check(snap, signals, "side stream")
        R.check_device_errors()
    finally:
        plan.close()
        bare.close()
    # a context created under SS_NO_GRAPH: the launches enqueued at every run, same bits
    ctx2 = ctypes.c_void_p()
    os.environ["SS_NO_GRAPH"] = "1"
    try:
        L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
    finally:
        del os.environ["SS_NO_GRAPH"]
    R2 = render.Renderer(R.device)
    R2.ctx = ctx2
    banks2 = [R2.rir_bank(to(c.h), direct_taps=taps) for c in cands]
    pool2 = R2.source_pool([render.MovingSource(to(c.x), bk, to(c.b), c.b) for c, bk in zip(cands, banks2)])
    dpool2 = R2.dry_pool(signals)
    sl2 = DrySlots(pool2, dpool2, cands, 7000, taps)
    plan2 = R2.plan_device(sl2.srcs, sl2.outs, direct_outs=sl2.douts)
    try:
        for a, b in ((sl2.picks, sl.picks), (sl2.dpicks, sl.dpicks), (sl2.starts, sl.starts)):
            a.copy_(b)
        plan2.run()
        assert not plan2.is_graph()
        snap = sl2.snap()
        torch.cuda.synchronize()
        sl.check(snap, signals, "no graph")
    finally:
        plan2.close()
        pool2.close()
        dpool2.close()
        for b in banks2:
            b.close()
        R2.lib.ss_destroy(ctx2)
    pool.close()
    dpool.close()


def test_refusals(world, draw_pools):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    cands, taps = world["speakers"]
    noi, _ = world["noise"]
    n_max = max(c.N for c in cands)
    signals = dry_signals(315, 3, n_max, 0)
    pool, npool, dpool = R.source_pool([c.src for c in cands]), R.source_pool([c.src for c in noi]), R.dry_pool(signals)
    short = R.dry_pool([s[:n_max - 1] for s in signals])
    hbanks = [R.rir_bank(c.h, host=True) for c in cands]
    hpool = R.source_pool([render.MovingSource(c.x, bk, c.b, c.b) for c, bk in zip(cands, hbanks)])
    gpool = R.source_pool([c.src for c in cands], lufs_targets=[-17.0] * len(cands))
    sp, _, dpool_lv, dry_dev, _, _ = draw_pools
    nolv = R.dry_pool(dry_dev)                               # long enough for sp, without level tables
    wl = 5000
    picks = torch.zeros(3, dtype=torch.int32, device="cuda")
    dpicks = torch.zeros(3, dtype=torch.int32, device="cuda")
    start = torch.zeros(1, dtype=torch.int32, device="cuda")
    u = torch.rand(11, dtype=torch.float64, device="cuda")
    used = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    outs = [torch.full((2, wl), NAN, device="cuda") for _ in range(3)]
    DP, PO = render.DryPick, render.Pooled

    def slots(p0=pool, d0=None, d1=None):
        return [PO(p0, picks[0], (start[0], wl), 0, d0), PO(pool, picks[1], (start[0], wl), 0, d1),
                PO(npool, picks[2], (start[0], wl))]

    def py(srcs, match, draws=None):
        with pytest.raises(ValueError, match=match):
            R.plan_device(srcs, outs, draws=draws)

    ctx2 = ctypes.c_void_p()
    L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
    R2 = render.Renderer(R.device)
    R2.ctx = ctx2
    foreign = R2.dry_pool(signals)
    closed = R.dry_pool(signals)
    closed.close()
    try:
        good = DP(dpool, dpicks[0])
        py(slots(p0=hpool, d0=good), "host pool")
        py(slots(p0=gpool, d0=good), "loudness gains")
        py(slots(d0=DP(short, dpicks[0])), "shorter than its pool's longest")
        py(slots(d0=DP(foreign, dpicks[0])), "another renderer's context")
        py(slots(d0=DP(closed, dpicks[0])), "is closed")
        py(slots(d0=DP(dpool, dpicks[0].cpu())), "dry pick of source 0")
        py(slots(d0=DP(dpool, dpicks[:2])), "dry pick of source 0")
        py([cands[0].src._replace(dry=good, window=(0, wl))] + slots()[1:], "not a pooled slot")
        # a draw speaker with a dry pick over a dry pool without tables (the pool's own tables do not count)
        dsrc = [PO(sp, picks[0], (start[0], LEN), 0, DP(dpool_lv, dpicks[0])), PO(sp, picks[1], (start[0], LEN))]
        douts = [torch.full((2, LEN), NAN, device="cuda") for _ in range(2)]
        with pytest.raises(ValueError, match="DryPool has no level tables"):
            R.plan_device([dsrc[0]._replace(dry=DP(nolv, dpicks[0])), dsrc[1]], douts,
                          draws=[render.CropDraw(start[0], [0, 1], u, used[0])])
        ok = R.plan_device(dsrc, douts, draws=[render.CropDraw(start[0], [0, 1], u, used[0])])
        ok.close()

        # the C ABI, past the Python checks
        srcs = slots(d0=good, d1=DP(dpool, dpicks[1]))
        items, n, keep = R._device_items(srcs, outs)
        arr = R._device_dry(srcs)
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_dry(R.ctx, items, n, None, 0, None, 0, arr, len(arr), ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)
        assert R.lib.ss_plan_create_dry(R.ctx, items, n, None, 0, None, 0, None, 0, ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)

        def c_call(picks_arr, n_picks=None, its=items, mixes=None, draws=None, want=L.SS_ERR_INVALID):
            h = ctypes.c_void_p()
            got = R.lib.ss_plan_create_dry(R.ctx, its, n, mixes, len(mixes) if mixes else 0, draws,
                                           len(draws) if draws else 0, picks_arr,
                                           len(picks_arr) if n_picks is None and picks_arr else (n_picks or 0),
                                           ctypes.byref(h))
            assert got == want and not h.value, (got, want)

        def one(**kw):
            a = (L.SsDryPick * 1)()
            a[0] = L.SsDryPick(slot=0, pool=dpool._h.value, pick_dev=dpicks[0].data_ptr())
            for k, v in kw.items():
                setattr(a[0], k, v)
            return a

        c_call(None, n_picks=1)                                  # NULL picks
        c_call(one(), n_picks=-1)
        c_call(one(slot=3))                                      # outside [0, n_items)
        c_call(one(slot=-1))
        two = (L.SsDryPick * 2)(one()[0], one()[0])
        c_call(two)                                              # one slot, two dry picks
        c_call(one(pool=None))
        c_call(one(pool=foreign._h.value))                       # another context
        c_call(one(pool=short._h.value))                         # a signal shorter than the longest candidate
        c_call(one(pick_dev=None))
        c_call(one(pick_dev=dpicks.data_ptr() + 2))              # unaligned
        its = (L.SsSource * n)()
        ctypes.memmove(its, items, ctypes.sizeof(L.SsSource) * n)
        fx, _, _ = R._device_items([cands[0].src._replace(window=(0, wl))], [outs[0]])
        its[0] = fx[0]
        c_call(one(), its=its)                                   # a slot that is not pooled
        its = (L.SsSource * n)()
        ctypes.memmove(its, items, ctypes.sizeof(L.SsSource) * n)
        its[0].pool = hpool._h.value
        c_call(one(), its=its)                                   # a host pool
        its[0].pool = gpool._h.value
        c_call(one(), its=its)                                   # a pool with gains
        # a dry pick over a range a mixture writes
        mix = torch.full((2, wl), NAN, device="cuda")
        sirs, snr = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
        mixes = R._device_mixes([render.Mixture([0, 1], [2], sirs, snr, mix)], outs, keep)
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_dry(R.ctx, items, n, mixes, 1, None, 0, one(), 1, ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)
        c_call(one(pick_dev=mix.data_ptr()), mixes=mixes)
        # a draw speaker with a dry pick over a dry pool without tables
        ditems, dn, dkeep = R._device_items(dsrc, douts)
        draws = R._device_draws([render.CropDraw(start[0], [0, 1], u, used[0])], dsrc, dkeep)
        h = ctypes.c_void_p()
        dl = (L.SsDryPick * 1)(L.SsDryPick(slot=0, pool=dpool_lv._h.value, pick_dev=dpicks[0].data_ptr()))
        assert R.lib.ss_plan_create_dry(R.ctx, ditems, dn, None, 0, draws, 1, dl, 1, ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)
        dl[0].pool = nolv._h.value
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_dry(R.ctx, ditems, dn, None, 0, draws, 1, dl, 1, ctypes.byref(h)) == \
            L.SS_ERR_INVALID and not h.value
        # ss_dry_pool_create
        x = (ctypes.c_void_p * 2)(signals[0].data_ptr(), signals[1].data_ptr())
        lens = np.array([signals[0].numel(), signals[1].numel()], np.int32)
        hp = ctypes.c_void_p()
        for args in ((R.ctx, x, lens.ctypes.data, 0, 0), (R.ctx, x, lens.ctypes.data, 2, 2),
                     (R.ctx, None, lens.ctypes.data, 2, 0), (R.ctx, x, None, 2, 0),
                     (R.ctx, (ctypes.c_void_p * 2)(x[0], None), lens.ctypes.data, 2, 0),
                     (R.ctx, (ctypes.c_void_p * 2)(x[0], x[1] + 2), lens.ctypes.data, 2, 0),
                     (R.ctx, x, np.array([5, 0], np.int32).ctypes.data, 2, 0),
                     (R.ctx, x, np.array([5, -3], np.int32).ctypes.data, 2, 0)):
            assert R.lib.ss_dry_pool_create(*args, ctypes.byref(hp)) == L.SS_ERR_INVALID and not hp.value, args
        torch.cuda.synchronize()
        for o in outs + douts + [mix]:
            assert torch.isnan(o).all()
        assert int(used[0]) == -7
    finally:
        foreign.close()
        R2.lib.ss_destroy(ctx2)
        for p in (pool, npool, dpool, short, hpool, gpool, nolv):
            p.close()
        for b in hbanks:
            b.close()


def test_training_scale():
    """16 examples x (2 dry-picked speakers + a dry-picked noise), 256 dry streams of 60 s with level tables, one
    CropDraw per example: the picked stems equal render_device, the starts equal draw_reference."""
    render, R = _R()
    rng = np.random.default_rng(331)
    spk = []
    for j in range(8):
        P, N = 4 + j % 3, 30 * RATE - 7001 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        spk.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    noi = [Cand(so.synth_dry(rng, 30 * RATE), so.synth_rirs(rng, 1, 2, 4096)[0], None) for _ in range(4)]
    g = torch.Generator(device="cuda")
    g.manual_seed(41)
    T = 60 * RATE
    dry = (torch.randn((256, T), generator=g, device="cuda") * 0.05)
    dry *= (torch.rand((256, T // 8000), generator=g, device="cuda") > 0.4).repeat_interleave(8000, 1)
    signals = list(dry.unbind(0))
    sp, npool = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])
    dpool = R.dry_pool(signals, levels=True)
    assert dpool.nbytes == 8 * 256 + 8 * 256 * (T + 1) + 8 * 256
    B = 16
    picks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    starts = torch.zeros(B, dtype=torch.int32, device="cuda")
    u = torch.zeros((B, 101), dtype=torch.float64, device="cuda")
    used = torch.zeros(B, dtype=torch.int32, device="cuda")
    sirs, snr = torch.zeros((B, 1), device="cuda"), torch.zeros(B, device="cuda")
    outs = [torch.empty((2, LEN), device="cuda") for _ in range(3 * B)]
    mix = torch.empty((B, LEN), device="cuda")
    srcs, mixtures, draws = [], [], []
    for b in range(B):
        for j, pl in enumerate((sp, sp, npool)):
            srcs.append(render.Pooled(pl, picks[b, j], (starts[b], LEN), 0, render.DryPick(dpool, dpicks[b, j])))
        mixtures.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sirs[b], snr[b], mix[b], mono=True))
        draws.append(render.CropDraw(starts[b], [3 * b, 3 * b + 1], u[b], used[b]))
    plan = R.plan_device(srcs, outs, mixtures=mixtures, draws=draws)
    try:
        checked = 0
        for run in range(2):
            picks[:, :2].copy_(torch.randint(0, len(spk), (B, 2), generator=g, device="cuda", dtype=torch.int32))
            picks[:, 2].copy_(torch.randint(0, len(noi), (B,), generator=g, device="cuda", dtype=torch.int32))
            dpicks.copy_(torch.randint(0, 256, (B, 3), generator=g, device="cuda", dtype=torch.int32))
            u.uniform_(generator=g)
            sirs.uniform_(-6, 6, generator=g)
            snr.uniform_(10, 20, generator=g)
            plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            for b in range(B):
                p = [int(v) for v in picks[b]]
                d = [int(v) for v in dpicks[b]]
                s, k = int(starts[b]), int(used[b])
                cs = (spk[p[0]], spk[p[1]], noi[p[2]])
                for j in range(3):
                    assert torch.equal(outs[3 * b + j], reference(cs[j], signals[d[j]], s, LEN, 0)[0]), (run, b, j)
                tabs = [dpool.level_table(d[0]).cpu().numpy(), dpool.level_table(d[1]).cpu().numpy()]
                Nr = [c.N for c in cs]
                ub = u[b].cpu().numpy()
                if dr.margins(tabs, [LEN, LEN], Nr, LEN, ub) < NEAR_DB:
                    continue
                assert (s, k) == dr.draw(tabs, [LEN, LEN], Nr, LEN, ub), (run, b)
                checked += 1
        assert checked >= 28
    finally:
        plan.close()
        for p in (sp, npool, dpool):
            p.close()
