"""Host dry pools (Renderer.dry_pool(..., host=True); ss_dry_pool_create with SS_DRY_HOST) through the real kernels.  A
host dry pool keeps its signals and level tables in pinned, mapped host memory; at every run k_stage copies the dry
samples each dry-picked slot's crop reads from the picked signal.  Checked:
  1. bits: for device and host source pools and for aligned speakers (k_render_fast) with direct stems, long RIRs
     (K > 1) and static noise, plans over a host dry pool equal the same plans over a device dry pool of the same signals
     and render_device of the picked candidate with the picked signal's first N samples; signals given as NumPy arrays,
     CPU and CUDA tensors, some exactly N long with N % 4 != 0, the others with NaN tails; mixtures over host-dry-picked
     slots of a device and a host pool equal ss_mix_dev on the plan's own stems;
  2. a host dry pool's level tables equal a device dry pool's bit for bit, and CropDraw over them gives the same starts,
     `used` and stems as over device tables, with speakers with and without dry picks in one draw;
  3. an out-of-range dry pick on a staged slot is clamped and reported as bit 4 (IndexError), then cleared;
  4. a device-pool plan launches exactly one kernel (k_stage) more per run than with a device dry pool, a host-pool plan
     as many as without dry picks; a run on a side stream behind queued work gives the same bits;
  5. nbytes counts the pointer arrays only, host_nbytes the padded arena and the tables, and device free memory does not
     drop by the signals' or the tables' size;
  6. refusals in Python and through the C ABI, with nothing written;
  7. one training-scale plan: 16 examples x (2 dry-picked speakers + a dry-picked noise) over 64 gappy 60 s streams, on
     device and host source pools, with draws and mixtures; every stem equals the device-dry-pool twin, and a sample of
     stems meets the float64 render reference (tests/render_reference.py) within its bounds."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from direct_path import direct_path_rirs
from draw_reference import gappy_dry
from gpu_plumbing import _R, _rms, to
from pool_worlds import DrawStep, DrySlots, _host_pool, _mix_dev, moving, noises, reference, speakers
from pool_worlds import draw_world  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

TAPS = 40
NAN = float("nan")
RATE = 16000
SLEEP = int(5e8)


@pytest.fixture(scope="module")
def world():
    spk = speakers(401, n=4, taps=TAPS)                       # aligned moving, direct sets
    lng = moving(402, [5000, 9000, 13000, 6000])              # K = 2, 3, 4, 2: grid, k_render<LONG>
    noi = noises(403, n=3)                                    # static
    out = {}
    for kind, cands, taps in (("speakers", spk, TAPS), ("long", lng, 0), ("noise", noi, 0)):
        render, R = _R()
        out[kind] = (cands, taps, {"device": R.source_pool([c.src for c in cands]),
                                   "host": _host_pool(R, render, cands, taps)})
    yield out
    for _, _, pools in out.values():
        for p in pools.values():
            p.close()


def signal_set(seed, n_max):
    """Five signals covering a pool whose longest candidate has n_max samples (n_max % 4 != 0): as given to the host dry
    pool (NumPy, CPU tensor, CUDA tensor) and as CUDA tensors for the device dry pool and the references.  Two are exactly
    n_max long, the others carry NaN tails no slot may read."""
    assert n_max % 4
    rng = np.random.default_rng(seed)
    arrays = []
    for tail in (0, 3001, 7, 0, 102):
        x = np.full(n_max + tail, np.nan, np.float32)
        x[:n_max] = so.synth_dry(rng, n_max)
        arrays.append(x)
    given = [arrays[0], torch.from_numpy(arrays[1].copy()), to(arrays[2]), torch.from_numpy(arrays[3].copy()),
             arrays[4]]
    return given, [to(a) for a in arrays]


def _twin(dst, src):
    for a, b in ((dst.picks, src.picks), (dst.dpicks, src.dpicks), (dst.starts, src.starts)):
        a.copy_(b)
    for o in dst.outs + (dst.douts or []):
        o.fill_(NAN)


@pytest.mark.parametrize("resident", ["device", "host"])
@pytest.mark.parametrize("kind", ["speakers", "long", "noise"])
def test_bits_equal_device_dry_pool_and_render_device(world, kind, resident):
    render, R = _R()
    cands, taps, pools = world[kind]
    pool, n_max = pools[resident], max(c.N for c in cands)
    given, cuda = signal_set(411, n_max)
    hdry = R.dry_pool(given, host=True)
    ddry = R.dry_pool(cuda)
    assert hdry.resident == "host" and hdry.n_min == n_max and hdry.sizes == [x.numel() for x in cuda]
    wl = 9000 if kind != "noise" else 20000
    sl = DrySlots(pool, hdry, cands, wl, taps)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    twin = None
    if resident == "device":                                  # a device dry pool only on a device pool's slots
        tw = DrySlots(pool, ddry, cands, wl, taps)
        twin = (tw, R.plan_device(tw.srcs, tw.outs, direct_outs=tw.douts))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(41)
    n_min = min(c.N for c in cands)
    try:
        snaps = []
        for run in range(6):
            sl.fill(gen, len(cands), hdry.n, n_min)
            if run == 0:                                      # the exactly-N signals at both ends of the longest candidate
                sl.picks.fill_(int(np.argmax([c.N for c in cands])))
                sl.dpicks.copy_(torch.tensor([0, 3, 0, 3], dtype=torch.int32))
                sl.starts.copy_(torch.tensor([0, n_max - wl, n_max - wl, 0], dtype=torch.int32))
            plan.run()
            snap = sl.snap()
            if twin:
                _twin(twin[0], sl)
                twin[1].run()
                tsnap = twin[0].snap()
                for a, b in zip(snap["outs"] + snap["douts"], tsnap["outs"] + tsnap["douts"]):
                    assert torch.equal(a, b), (kind, run)
            snaps.append(snap)
        assert plan.is_graph()
        torch.cuda.synchronize()
        R.check_device_errors()
        for r, snap in enumerate(snaps):
            sl.check(snap, cuda, "%s %s run %d" % (kind, resident, r))
    finally:
        plan.close()
        if twin:
            twin[1].close()
        hdry.close()
        ddry.close()


def test_mixtures_over_host_dry_picks(world):
    render, R = _R()
    spk, _, spools = world["speakers"]
    noi, _, npools = world["noise"]
    given, cuda = signal_set(412, max(c.N for c in spk + noi) | 1)
    hdry = R.dry_pool(given, host=True)
    sp, npool = spools["device"], npools["host"]              # a device pool's and a host pool's slots, one dry pool
    wl, B = 12000, 3
    picks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((B, 3), dtype=torch.int32, device="cuda")
    starts = torch.zeros(B, dtype=torch.int32, device="cuda")
    sirs, snr = torch.zeros((B, 1), device="cuda"), torch.zeros(B, device="cuda")
    outs = [torch.empty((2, wl), device="cuda") for _ in range(3 * B)]
    mix, spo = torch.empty((B, 2, wl), device="cuda"), torch.empty((B, 2, 2, wl), device="cuda")
    srcs, mixtures = [], []
    for b in range(B):
        for j, pl in enumerate((sp, sp, npool)):
            srcs.append(render.Pooled(pl, picks[b, j], (starts[b], wl), 0, render.DryPick(hdry, dpicks[b, j])))
        mixtures.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sirs[b], snr[b], mix[b], spo[b]))
    plan = R.plan_device(srcs, outs, mixtures=mixtures)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(42)
    n_min = min(c.N for c in spk + noi)
    try:
        for run in range(3):
            picks[:, :2].copy_(torch.randint(0, len(spk), (B, 2), generator=gen, device="cuda", dtype=torch.int32))
            picks[:, 2].copy_(torch.randint(0, len(noi), (B,), generator=gen, device="cuda", dtype=torch.int32))
            dpicks.copy_(torch.randint(0, hdry.n, (B, 3), generator=gen, device="cuda", dtype=torch.int32))
            starts.copy_(torch.randint(0, n_min - wl + 1, (B,), generator=gen, device="cuda", dtype=torch.int32))
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(10, 20, generator=gen)
            plan.run()
            torch.cuda.synchronize()
            for b in range(B):
                for j, cs in enumerate((spk, spk, noi)):
                    c = cs[int(picks[b, j])]
                    ref, _ = reference(c, cuda[int(dpicks[b, j])], int(starts[b]), wl, 0)
                    assert torch.equal(outs[3 * b + j], ref), (run, b, j)
                m, s = _mix_dev(R, torch.stack([outs[3 * b].reshape(-1), outs[3 * b + 1].reshape(-1)]),
                                outs[3 * b + 2].reshape(1, -1), sirs[b], snr[b])
                assert torch.equal(mix[b].reshape(-1), m) and torch.equal(spo[b].reshape(2, -1), s), (run, b)
        R.check_device_errors()
    finally:
        plan.close()
        hdry.close()


def test_tables_and_draws_equal_device_tables(draw_world):
    render, R = _R()
    spk, noi, dry = draw_world
    sp = R.source_pool([c.src for c in spk], levels="mono")
    npool = R.source_pool([c.src for c in noi])
    hdry = R.dry_pool(dry, levels=True, host=True)            # NumPy signals
    ddry = R.dry_pool([to(x) for x in dry], levels=True)
    try:
        for i in range(hdry.n):
            assert torch.equal(hdry.level_table(i), ddry.level_table(i)), i
        assert hdry.level_table(hdry.n) is None
        for mixed in (True, False):
            hs = DrawStep(R, render, sp, npool, hdry, B=12, mixed=mixed)
            ds = DrawStep(R, render, sp, npool, ddry, B=12, mixed=mixed)
            gen = torch.Generator(device="cuda")
            gen.manual_seed(43 + mixed)
            try:
                for run in range(6):
                    hs.fill(gen, len(spk), len(noi), hdry.n)
                    for a, b in ((ds.picks, hs.picks), (ds.dpicks, hs.dpicks), (ds.u, hs.u)):
                        a.copy_(b)
                    hs.plan.run()
                    ds.plan.run()
                    torch.cuda.synchronize()
                    assert torch.equal(hs.starts, ds.starts) and torch.equal(hs.used, ds.used), (mixed, run)
                    for a, b in zip(hs.outs, ds.outs):
                        assert torch.equal(a, b), (mixed, run)
                R.check_device_errors()
            finally:
                hs.plan.close()
                ds.plan.close()
    finally:
        for p in (sp, npool, hdry, ddry):
            p.close()


@pytest.mark.parametrize("resident", ["device", "host"])
def test_clamped_dry_pick_on_a_staged_slot(world, resident):
    render, R = _R()
    cands, taps, pools = world["speakers"]
    given, cuda = signal_set(413, max(c.N for c in cands))
    hdry = R.dry_pool(given[:3], host=True)
    sl = DrySlots(pools[resident], hdry, cands, 5000, taps, k=2)
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
            R.check_device_errors()                          # reported once, then cleared
            snap = sl.snap()
            snap["dpicks"][0] = want
            sl.check(snap, cuda, "clamped %d" % bad)
    finally:
        plan.close()
        hdry.close()


def _count(R, plan):
    plan.run()
    c0 = R.launch_count()
    plan.run()
    return R.launch_count() - c0


def test_launches_and_side_stream(world):
    render, R = _R()
    cands, taps, pools = world["speakers"]
    given, cuda = signal_set(414, max(c.N for c in cands))
    hdry, ddry = R.dry_pool(given, host=True), R.dry_pool(cuda)
    n_min = min(c.N for c in cands)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(44)
    plans = []
    try:
        sets = {}
        for name, pool, dpool, dry in (("dev+host", pools["device"], hdry, True), ("dev+dev", pools["device"], ddry, True),
                                       ("host+host", pools["host"], hdry, True), ("host", pools["host"], hdry, False)):
            sl = DrySlots(pool, dpool, cands, 7000, taps, dry=dry)
            plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
            plans.append(plan)
            sl.fill(gen, len(cands), hdry.n, n_min)
            sets[name] = (sl, plan, _count(R, plan))
            assert plan.is_graph()
        assert sets["dev+host"][2] == sets["dev+dev"][2] + 1        # k_stage
        assert sets["host+host"][2] == sets["host"][2]              # k_stage runs anyway
        # a side stream behind queued work, with the picks written on it
        for name in ("dev+host", "host+host"):
            sl, plan, _ = sets[name]
            plan.run()
            ref = [o.clone() for o in sl.outs + sl.douts]
            torch.cuda.synchronize()
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                keep = (sl.picks.clone(), sl.dpicks.clone(), sl.starts.clone())
                for o in sl.outs + sl.douts:
                    o.fill_(NAN)
                sl.dpicks.fill_(0)
                torch.cuda._sleep(SLEEP)
                for a, b in zip((sl.picks, sl.dpicks, sl.starts), keep):
                    a.copy_(b)
                plan.run(stream=s.cuda_stream)
                busy = not s.query()
            assert busy
            s.synchronize()
            for a, b in zip(ref, sl.outs + sl.douts):
                assert torch.equal(a, b), name
            sl.check(sl.snap(), cuda, name + " side stream")
        R.check_device_errors()
    finally:
        for p in plans:
            p.close()
        hdry.close()
        ddry.close()


def test_memory():
    _, R = _R()
    rng = np.random.default_rng(415)
    lens = [int(v) for v in rng.integers(1, 40, 9)] + [1, 5, 4097]
    small = [so.synth_dry(rng, n) for n in lens]
    for levels in (False, True):
        p = R.dry_pool(small, levels=levels, host=True)
        try:
            n = len(small)
            assert p.nbytes == 8 * n + (8 * n if levels else 0)
            arena = sum((4 * k + 63) // 64 * 64 for k in lens)
            assert p.host_nbytes == arena + (8 * sum(k + 1 for k in lens) if levels else 0)
            if levels:
                for i, x in enumerate(small):
                    q = p.level_table(i).cpu().numpy()
                    assert q.shape == (len(x) + 1,) and q[0] == 0.0
        finally:
            p.close()
    # 48 signals of 4 M samples: 768 MB of signal and 1.5 GB of tables stay in host memory
    big = [np.full(1 << 22, 0.25, np.float32) for _ in range(48)]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    p = R.dry_pool(big, levels=True, host=True)
    try:
        free1 = torch.cuda.mem_get_info()[0]
        assert free0 - free1 < 64 << 20, (free0 - free1) / 2 ** 20
        assert p.host_nbytes == 48 * (4 << 22) + 48 * 8 * ((1 << 22) + 1)
        q = p.level_table(47)
        assert float(q[-1]) == 0.0625 * (1 << 22) and float(q[1]) == 0.0625
    finally:
        p.close()


def test_refusals(world):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    cands, taps, pools = world["speakers"]
    dpool_, hpool = pools["device"], pools["host"]
    n_max = max(c.N for c in cands)
    given, cuda = signal_set(416, n_max)
    hdry = R.dry_pool(given, host=True)
    ddry = R.dry_pool(cuda)
    short = R.dry_pool([x[:n_max - 1] for x in cuda], host=True)
    gpool = R.source_pool([c.src for c in cands], lufs_targets=[-17.0] * len(cands))
    ctx2 = ctypes.c_void_p()
    L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
    R2 = render.Renderer(R.device)
    R2.ctx = ctx2
    foreign = R2.dry_pool(given, host=True)
    closed = R.dry_pool(given, host=True)
    closed.close()
    wl = 5000
    picks = torch.zeros(2, dtype=torch.int32, device="cuda")
    dpicks = torch.zeros(2, dtype=torch.int32, device="cuda")
    start = torch.zeros(1, dtype=torch.int32, device="cuda")
    outs = [torch.full((2, wl), NAN, device="cuda") for _ in range(2)]
    DP, PO = render.DryPick, render.Pooled

    def slots(p0, d0):
        return [PO(p0, picks[0], (start[0], wl), 0, d0), PO(dpool_, picks[1], (start[0], wl))]

    def py(srcs, match):
        with pytest.raises(ValueError, match=match):
            R.plan_device(srcs, outs)

    try:
        for p0 in (dpool_, hpool):
            py(slots(p0, DP(short, dpicks[0])), "shorter than its pool's longest")
            py(slots(p0, DP(foreign, dpicks[0])), "another renderer's context")
            py(slots(p0, DP(closed, dpicks[0])), "is closed")
        py(slots(gpool, DP(hdry, dpicks[0])), "loudness gains")
        py(slots(hpool, DP(ddry, dpicks[0])), "host pool")          # a device dry pool on a host pool's slot
        for bad in (np.zeros((2, n_max), np.float32), np.zeros(0, np.float32), torch.zeros((2, n_max)),
                    torch.zeros((2, n_max), device="cuda"), torch.zeros(0, device="cuda")):
            with pytest.raises(ValueError, match="1-D and not empty"):
                R.dry_pool([given[0], bad], host=True)
        with pytest.raises(ValueError, match="1 to 2\\^24 signals"):
            R.dry_pool([], host=True)

        # the C ABI, past the Python checks
        for p0 in (dpool_, hpool):
            srcs = slots(p0, DP(hdry, dpicks[0]))
            items, n, keep = R._device_items(srcs, outs)
            arr = R._device_dry(srcs)
            h = ctypes.c_void_p()
            assert R.lib.ss_plan_create_dry(R.ctx, items, n, None, 0, None, 0, arr, 1, ctypes.byref(h)) == 0
            R.lib.ss_plan_destroy(h)
            for dp in (short, foreign, ddry) if p0 is hpool else (short, foreign):
                bad = (L.SsDryPick * 1)(L.SsDryPick(slot=0, pool=dp._h.value, pick_dev=dpicks[0].data_ptr()))
                h = ctypes.c_void_p()
                assert R.lib.ss_plan_create_dry(R.ctx, items, n, None, 0, None, 0, bad, 1, ctypes.byref(h)) == \
                    L.SS_ERR_INVALID and not h.value, dp
        its = (L.SsSource * n)()
        ctypes.memmove(its, items, ctypes.sizeof(L.SsSource) * n)
        its[0].pool = gpool._h.value
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_dry(R.ctx, its, n, None, 0, None, 0, arr, 1, ctypes.byref(h)) == \
            L.SS_ERR_INVALID and not h.value
        # ss_dry_pool_create with SS_DRY_HOST over host pointers
        a = [np.ascontiguousarray(x[:100], np.float32) for x in given[:2] if isinstance(x, np.ndarray)] * 2
        x = (ctypes.c_void_p * 2)(a[0].ctypes.data, a[1].ctypes.data)
        lens = np.array([100, 100], np.int32)
        H = L.SS_DRY_HOST
        hp = ctypes.c_void_p()
        assert R.lib.ss_dry_pool_create(R.ctx, x, lens.ctypes.data, 2, H | L.SS_DRY_LEVELS, ctypes.byref(hp)) == 0
        assert R.lib.ss_dry_pool_host_bytes(hp) == 2 * 448 + 2 * 808 and R.lib.ss_dry_pool_bytes(hp) == 32
        R.lib.ss_dry_pool_destroy(hp)
        hp = ctypes.c_void_p()
        for args in ((R.ctx, x, lens.ctypes.data, 0, H), (R.ctx, x, lens.ctypes.data, 2, H | 0x200),
                     (R.ctx, None, lens.ctypes.data, 2, H), (R.ctx, x, None, 2, H),
                     (R.ctx, (ctypes.c_void_p * 2)(x[0], None), lens.ctypes.data, 2, H),
                     (R.ctx, (ctypes.c_void_p * 2)(x[0], x[1] + 2), lens.ctypes.data, 2, H),
                     (R.ctx, x, np.array([5, 0], np.int32).ctypes.data, 2, H),
                     (R.ctx, x, np.array([5, -3], np.int32).ctypes.data, 2, H)):
            assert R.lib.ss_dry_pool_create(*args, ctypes.byref(hp)) == L.SS_ERR_INVALID and not hp.value, args
        assert R.lib.ss_dry_pool_host_bytes(None) == 0 and R.lib.ss_dry_pool_host_bytes(ddry._h) == 0
        torch.cuda.synchronize()
        for o in outs:
            assert torch.isnan(o).all()
    finally:
        foreign.close()
        R2.lib.ss_destroy(ctx2)
        for p in (hdry, ddry, short, gpool):
            p.close()


# ------------------------------------------------------------------------------------------------ training scale
LEN, U, S = 4 * RATE, 16, 2


def test_training_scale(draw_world):
    """16 examples x (2 speakers + noise), every slot dry-picked from 64 gappy streams of 60 s held in host memory, one
    CropDraw over the dry tables and one mixture per example, on device and on host source pools.  Every stem, mixture,
    start and `used` equals the twin plan over a device dry pool and device pools; 8 stems per run meet float64."""
    render, R = _R()
    spk, noi, _ = draw_world
    rng = np.random.default_rng(417)
    streams = [gappy_dry(rng, 60 * RATE) for _ in range(64)]
    hdry = R.dry_pool(streams, levels=True, host=True)
    ddry = R.dry_pool([to(x) for x in streams], levels=True)
    assert hdry.nbytes == 2 * 8 * 64 and ddry.nbytes == 8 * 64 + 8 * 64 * (60 * RATE + 1) + 8 * 64
    pools = {"device": (R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])),
             "host": (_host_pool(R, render, spk), _host_pool(R, render, noi))}
    twin_pools = pools["device"]
    picks = torch.zeros((U, S + 1), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((U, S + 1), dtype=torch.int32, device="cuda")
    u = torch.zeros((U, 101), dtype=torch.float64, device="cuda")
    sirs, snr = torch.zeros((U, S - 1), device="cuda"), torch.zeros(U, device="cuda")

    def build(sp, npool, dpool):
        starts = torch.zeros(U, dtype=torch.int32, device="cuda")
        used = torch.zeros(U, dtype=torch.int32, device="cuda")
        outs = [torch.full((2, LEN), NAN, device="cuda") for _ in range(U * (S + 1))]
        mix, spo = torch.empty((U, 2, LEN), device="cuda"), torch.empty((U, S, 2, LEN), device="cuda")
        srcs, mixes, draws = [], [], []
        for e in range(U):
            for j, pl in enumerate((sp,) * S + (npool,)):
                srcs.append(render.Pooled(pl, picks[e, j], (starts[e], LEN), 0, render.DryPick(dpool, dpicks[e, j])))
            k = (S + 1) * e
            mixes.append(render.Mixture(list(range(k, k + S)), [k + S], sirs[e], snr[e], mix[e], spo[e]))
            draws.append(render.CropDraw(starts[e], list(range(k, k + S)), u[e], used[e]))
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), dict(starts=starts, used=used, outs=outs,
                                                                             mix=mix, spo=spo)

    twin, tw = build(twin_pools[0], twin_pools[1], ddry)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(47)
    worst = [0.0, 0.0]
    checked = 0
    try:
        for resident in ("device", "host"):
            plan, st = build(pools[resident][0], pools[resident][1], hdry)
            try:
                for run in range(3):
                    picks[:, :S].copy_(torch.randint(0, len(spk), (U, S), generator=gen, device="cuda", dtype=torch.int32))
                    picks[:, S].copy_(torch.randint(0, len(noi), (U,), generator=gen, device="cuda", dtype=torch.int32))
                    dpicks.copy_(torch.randint(0, hdry.n, (U, S + 1), generator=gen, device="cuda", dtype=torch.int32))
                    u.uniform_(generator=gen)
                    sirs.uniform_(-6, 6, generator=gen)
                    snr.uniform_(10, 20, generator=gen)
                    plan.run()
                    twin.run()
                    torch.cuda.synchronize()
                    for key in ("starts", "used", "mix", "spo"):
                        assert torch.equal(st[key], tw[key]), (resident, run, key)
                    for a, b in zip(st["outs"], tw["outs"]):
                        assert torch.isfinite(a).all() and torch.equal(a, b), (resident, run)
                    # a sample of stems against float64: render_f64 of the picked signal's first N samples
                    P_, D_, T_ = picks.cpu().numpy(), dpicks.cpu().numpy(), st["starts"].cpu().numpy()
                    for q in range(8):
                        e, j = (run * 5 + q * 3) % U, q % (S + 1)
                        c = (spk if j < S else noi)[int(P_[e, j])]
                        x = streams[int(D_[e, j])][:c.N]
                        a = int(T_[e])
                        y = st["outs"][(S + 1) * e + j].cpu().numpy()
                        y64, scale = render_check_inputs(x, c.h, 1 if c.b is not None else 0, bounds=c.b,
                                                         window=(a, LEN))
                        quiet = _rms(y64) < _rms(scale) / 32
                        w, g = check_render(y, y64, scale, TAU_LOCAL, np.inf if quiet else TAU_GLOBAL, n0=a,
                                            label="%s run %d ex %d stem %d" % (resident, run, e, j))
                        if quiet:
                            g = _rms(np.asarray(y, np.float64) - y64) / _rms(scale)
                            assert g <= TAU_GLOBAL, (resident, run, e, j, g)
                        worst = [max(worst[0], w), max(worst[1], g)]
                        checked += 1
                R.check_device_errors()
            finally:
                plan.close()
        print("\nhost dry pool, training scale: %d stems against float64, worst per-sample ratio %.3g (bound %.3g), "
              "worst global relative RMS %.3g (bound %.3g)" % (checked, worst[0], TAU_LOCAL, worst[1], TAU_GLOBAL))
    finally:
        twin.close()
        for pair in pools.values():
            for p in pair:
                p.close()
        hdry.close()
        ddry.close()


def test_direct_stems_of_a_host_pool_against_float64(world):
    """Direct stems of a host pool's slots with host dry picks against the float64 render of the direct-path RIRs."""
    render, R = _R()
    cands, taps, pools = world["speakers"]
    given, cuda = signal_set(418, max(c.N for c in cands))
    hdry = R.dry_pool(given, host=True)
    sl = DrySlots(pools["host"], hdry, cands, 6000, taps, k=2)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    try:
        sl.picks.copy_(torch.tensor([0, 3], dtype=torch.int32))
        sl.dpicks.copy_(torch.tensor([2, 4], dtype=torch.int32))
        sl.starts.copy_(torch.tensor([1234, 20001], dtype=torch.int32))
        plan.run()
        torch.cuda.synchronize()
        for j in range(2):
            c = cands[int(sl.picks[j])]
            x = cuda[int(sl.dpicks[j])][:c.N].cpu().numpy()
            a = int(sl.starts[j])
            y64, scale = render_check_inputs(x, direct_path_rirs(c.h, TAPS), 1, bounds=c.b, window=(a, 6000))
            check_render(sl.douts[j].cpu().numpy(), y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=a, label="direct %d" % j)
    finally:
        plan.close()
        hdry.close()
