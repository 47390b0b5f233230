"""16-bit dry pools (Renderer.dry_pool(..., dtype="int16"); ss_dry_pool_create_i16) through the real kernels.  Every plan
is built twice, once over a float32 dry pool and once over a 16-bit pool of the same values k / 32768, and both are run
on the same picks, starts, SIRs, SNRs and variates.  Checked, bit for bit:
  1. stems and direct stems over the aligned k_render_fast pool (direct sets), a grid pool (K = 3), a mixed-length
     long-RIR pool (K = 2..4) and static noise, for device and host source pools crossed with device and host 16-bit
     pools (a float dry pool on a host pool's slots is a host one), over several runs with changing picks and no host
     synchronisation, one of them on a side stream behind queued work;
  2. training steps with start draws (a 16-bit and a float speaker in every draw), mixtures per channel and mono,
     speakers_out, rms_db, drawn starts and `used`;
  3. pair gains: the (LUFS, gain) table and the stems of pair-gained slots;
  4. level_table(i) against the float pool's, the sparse table itself, and level_stride;
  5. nbytes / host_nbytes against the formulas of include/sonicsim_b200.h;
  6. clamped dry picks report bit 4 (IndexError) on both arms, with the same stems;
  7. refusals in Python and through the C ABI, with no pool created."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from gpu_plumbing import _R
from pool_worlds import DrySlots, _host_pool, longs, moving, noises, speakers

pytestmark = pytest.mark.gpu

TAPS = 40
NAN = float("nan")
RATE = 16000
SLEEP = int(5e8)


def gappy_i16(rng, N, burst=(0.2, 1.0), gap=(0.0, 1.5)):
    """create_long_audio's layout in int16: silence, a burst of speech-like noise at a random level, silence, ..."""
    k = np.zeros(N, np.int16)
    pos = int(rng.integers(0, int(gap[1] * RATE)))
    while pos < N:
        n = int(rng.integers(int(burst[0] * RATE), int(burst[1] * RATE)))
        m = min(n, N - pos)
        v = so.synth_dry(rng, n)[:m].astype(np.float64)
        v *= rng.uniform(0.05, 0.9) / max(1e-9, np.abs(v).max())
        k[pos:pos + m] = np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16)
        pos += n + int(rng.integers(int(gap[0] * RATE), int(gap[1] * RATE)))
    return k


def values(k):
    return k.astype(np.float32) / np.float32(32768)


def i16_signals(seed, n, n_max, **kw):
    """n int16 signals of at least n_max samples (different lengths, N % 4 != 0 for some)."""
    rng = np.random.default_rng(seed)
    return [gappy_i16(rng, n_max + int(t), **kw) for t in rng.integers(0, 5000, n)]


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    kinds = {"aligned": (speakers(601, n=4, taps=TAPS), TAPS), "grid": (longs(602), 0),
             "mixedK": (moving(603, [5000, 9000, 13000, 6000]), 0), "noise": (noises(604, n=3), 0)}
    out = {}
    for kind, (cands, taps) in kinds.items():
        out[kind] = (cands, taps, {"device": R.source_pool([c.src for c in cands]),
                                   "host": _host_pool(R, render, cands, taps)})
    yield out
    for _, _, pools in out.values():
        for p in pools.values():
            p.close()


def twin_pools(R, ks, src_resident, i16_resident, levels=False):
    """The float arm's dry pool (host when the source pool is: a device float pool cannot serve a host pool's slots)
    and the 16-bit pool, over the same values; the 16-bit pool's signals given as int16 NumPy, CPU and CUDA tensors and
    float arrays on the grid."""
    fl = [values(k) for k in ks]
    given = []
    for j, k in enumerate(ks):
        given.append([k, torch.from_numpy(k.copy()), torch.from_numpy(k.copy()).cuda(), fl[j],
                      torch.from_numpy(fl[j].copy()).cuda()][j % 5])
    if src_resident == "host":
        fpool = R.dry_pool(fl, levels=levels, host=True)
    else:
        fpool = R.dry_pool([torch.from_numpy(x).cuda() for x in fl], levels=levels)
    ipool = R.dry_pool(given, levels=levels, host=i16_resident == "host", dtype="int16")
    assert ipool.dtype == "int16" and ipool.level_stride == 64 and ipool.resident == i16_resident
    assert ipool.sizes == fpool.sizes and ipool.signals == []
    return fpool, ipool


def _copy_inputs(dst, src):
    for a, b in ((dst.picks, src.picks), (dst.dpicks, src.dpicks), (dst.starts, src.starts)):
        a.copy_(b)
    for o in dst.outs + (dst.douts or []):
        o.fill_(NAN)


# ------------------------------------------------------------------------------------------------------ 1. stems
@pytest.mark.parametrize("i16_resident", ["device", "host"])
@pytest.mark.parametrize("src_resident", ["device", "host"])
@pytest.mark.parametrize("kind", ["aligned", "grid", "mixedK", "noise"])
def test_stems_equal_the_float_pool(world, kind, src_resident, i16_resident):
    render, R = _R()
    cands, taps, pools = world[kind]
    pool, n_max = pools[src_resident], max(c.N for c in cands)
    ks = i16_signals(611, 5, n_max)
    fpool, ipool = twin_pools(R, ks, src_resident, i16_resident)
    wl = min(9000, min(c.N for c in cands) - 1) if kind != "noise" else 20000
    A, Bs = DrySlots(pool, fpool, cands, wl, taps), DrySlots(pool, ipool, cands, wl, taps)
    pa = R.plan_device(A.srcs, A.outs, direct_outs=A.douts)
    pb = R.plan_device(Bs.srcs, Bs.outs, direct_outs=Bs.douts)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(61)
    n_min = min(c.N for c in cands)
    side = torch.cuda.Stream()
    try:
        snaps = []
        for run in range(6):
            A.fill(gen, len(cands), fpool.n, n_min)
            if run == 0:                                  # both ends of the longest candidate
                A.picks.fill_(int(np.argmax([c.N for c in cands])))
                A.starts.copy_(torch.tensor([0, n_max - wl, n_max - wl, 0], dtype=torch.int32))
            _copy_inputs(Bs, A)
            if run == 4:                                  # on a side stream behind queued work
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    torch.cuda._sleep(SLEEP)
                    pa.run(stream=side.cuda_stream)
                    pb.run(stream=side.cuda_stream)
                    busy = not side.query()
                    snaps.append((A.snap(), Bs.snap()))
                torch.cuda.current_stream().wait_stream(side)
                assert busy
                continue
            pa.run()
            pb.run()
            snaps.append((A.snap(), Bs.snap()))
        assert pa.is_graph() and pb.is_graph()
        torch.cuda.synchronize()
        R.check_device_errors()
        pairs = set()
        for r, (a, b) in enumerate(snaps):
            for x, y in zip(a["outs"] + a["douts"], b["outs"] + b["douts"]):
                assert torch.isfinite(x).all() and torch.equal(x, y), (kind, run, r)
            pairs |= {(int(p), int(d)) for p, d in zip(a["picks"], a["dpicks"])}
        assert len(pairs) >= 8
        # and against render_device of the picked candidate with the float values, for the first run
        A.check(snaps[0][0], [torch.from_numpy(values(k)).cuda() for k in ks], "%s reference" % kind)
    finally:
        pa.close()
        pb.close()
        fpool.close()
        ipool.close()


# ------------------------------------------------------------------------------------------- 2. draws and mixtures
LEN = RATE


class Step:
    """B examples: speaker 0 dry-picked from `dpool` (the arm's pool), speaker 1 from `fshared` (a float pool with
    tables, the same in both arms), a noise dry-picked from `dpool`; one CropDraw over both speakers, one mixture per
    channel and one mono."""

    def __init__(self, R, render, sp, npool, dpool, fshared, B, thr=-40.0, tries=37):
        d = "cuda"
        self.B = B
        self.picks = torch.zeros((B, 3), dtype=torch.int32, device=d)
        self.dpicks = torch.zeros((B, 3), dtype=torch.int32, device=d)
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.u = torch.zeros((B, tries), dtype=torch.float64, device=d)
        self.used = torch.full((B,), -7, dtype=torch.int32, device=d)
        self.sirs = torch.zeros((B, 1), device=d)
        self.snr = torch.zeros(B, device=d)
        self.outs = [torch.empty((2, LEN), device=d) for _ in range(3 * B)]
        self.mix = torch.empty((B, 2, LEN), device=d)
        self.spo = torch.empty((B, 2, 2, LEN), device=d)
        self.rms = torch.empty((B, 2), device=d)
        self.mmix = torch.empty((B, LEN), device=d)
        self.mspo = torch.empty((B, 2, LEN), device=d)
        self.mrms = torch.empty((B, 2), device=d)
        srcs, draws, mixes = [], [], []
        for b in range(B):
            w = (self.starts[b], LEN)
            srcs += [render.Pooled(sp, self.picks[b, 0], w, 0, render.DryPick(dpool, self.dpicks[b, 0])),
                     render.Pooled(sp, self.picks[b, 1], w, 0, render.DryPick(fshared, self.dpicks[b, 1])),
                     render.Pooled(npool, self.picks[b, 2], w, 0, render.DryPick(dpool, self.dpicks[b, 2]))]
            draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], self.u[b], self.used[b], thr))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mix[b],
                                        self.spo[b], self.rms[b]))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mmix[b],
                                        self.mspo[b], self.mrms[b], mono=True))
        self.plan = R.plan_device(srcs, self.outs, mixtures=mixes, draws=draws)

    def fill(self, gen, ns, nn, nd, nf):
        B = self.B
        self.picks[:, :2].copy_(torch.randint(0, ns, (B, 2), generator=gen, device="cuda", dtype=torch.int32))
        self.picks[:, 2].copy_(torch.randint(0, nn, (B,), generator=gen, device="cuda", dtype=torch.int32))
        self.dpicks[:, 0].copy_(torch.randint(0, nd, (B,), generator=gen, device="cuda", dtype=torch.int32))
        self.dpicks[:, 1].copy_(torch.randint(0, nf, (B,), generator=gen, device="cuda", dtype=torch.int32))
        self.dpicks[:, 2].copy_(torch.randint(0, nd, (B,), generator=gen, device="cuda", dtype=torch.int32))
        self.u.uniform_(generator=gen)
        self.sirs.uniform_(-6, 6, generator=gen)
        self.snr.uniform_(5, 20, generator=gen)

    def copy_from(self, o):
        for a, b in ((self.picks, o.picks), (self.dpicks, o.dpicks), (self.u, o.u), (self.sirs, o.sirs),
                     (self.snr, o.snr)):
            a.copy_(b)

    def results(self):
        for t in self.outs + [self.mix, self.spo, self.rms, self.mmix, self.mspo, self.mrms]:
            yield t
        yield self.starts
        yield self.used

    def clear(self):
        for t in self.outs + [self.mix, self.spo, self.rms, self.mmix, self.mspo, self.mrms]:
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)


@pytest.mark.parametrize("i16_resident", ["device", "host"])
@pytest.mark.parametrize("src_resident", ["device", "host"])
def test_draws_and_mixtures_equal_the_float_pool(world, src_resident, i16_resident):
    render, R = _R()
    spk, _, spools = world["aligned"]
    noi, _, npools = world["noise"]
    n_max = max(c.N for c in spk + noi)
    ks = i16_signals(621, 6, n_max, burst=(0.2, 0.8), gap=(0.5, 2.5))     # many crops wholly in a gap
    fpool, ipool = twin_pools(R, ks, src_resident, i16_resident, levels=True)
    rng = np.random.default_rng(622)
    shared = [values(gappy_i16(rng, n_max + 17, burst=(0.2, 0.8), gap=(0.5, 2.5))) for _ in range(3)]
    fshared = R.dry_pool(shared, levels=True, host=True)
    B = 12
    A = Step(R, render, spools[src_resident], npools[src_resident], fpool, fshared, B)
    Bs = Step(R, render, spools[src_resident], npools[src_resident], ipool, fshared, B)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(62)
    try:
        snaps = []
        for run in range(6):
            A.fill(gen, len(spk), len(noi), fpool.n, fshared.n)
            Bs.copy_from(A)
            A.clear()
            Bs.clear()
            A.plan.run()
            Bs.plan.run()
            snaps.append(([t.clone() for t in A.results()], [t.clone() for t in Bs.results()]))
        torch.cuda.synchronize()
        R.check_device_errors()
        outcomes = set()
        for r, (a, b) in enumerate(snaps):
            for j, (x, y) in enumerate(zip(a, b)):
                assert torch.equal(x, y), (run, r, j)
            outcomes |= {"first" if v == 1 else "later" if v > 1 else "none" for v in a[-1].cpu().numpy()}
            assert (a[-2] >= 0).all()
        assert "later" in outcomes and "first" in outcomes, outcomes     # silent crops were rejected
    finally:
        for p in (A.plan, Bs.plan, fpool, ipool, fshared):
            p.close()


# --------------------------------------------------------------------------------------------------- 3. pair gains
@pytest.mark.parametrize("i16_resident", ["device", "host"])
@pytest.mark.parametrize("src_resident", ["device", "host"])
def test_pair_gains_equal_the_float_pool(world, src_resident, i16_resident):
    render, R = _R()
    cands, taps, pools = world["aligned"]
    pool = pools[src_resident]
    ks = i16_signals(631, 3, max(c.N for c in cands))
    fpool, ipool = twin_pools(R, ks, src_resident, i16_resident)
    t = np.random.default_rng(632).uniform(-19, -15, (3, len(cands)))
    t[1, 2] = NAN
    ga = R.pair_gains(pool, fpool, t, sr=RATE)
    gb = R.pair_gains(pool, ipool, t, sr=RATE)
    la, lb = ga.loudness, gb.loudness
    assert np.array_equal(np.isnan(la), np.isnan(lb)) and np.array_equal(la[~np.isnan(la)], lb[~np.isnan(lb)])
    assert ga.nbytes == gb.nbytes == 4 * 3 * len(cands)
    wl = 9000
    A = DrySlots(pool, fpool, cands, wl, taps)
    Bs = DrySlots(pool, ipool, cands, wl, taps)
    A.srcs = [s._replace(dry=s.dry._replace(gains=ga)) for s in A.srcs]
    Bs.srcs = [s._replace(dry=s.dry._replace(gains=gb)) for s in Bs.srcs]
    pa = R.plan_device(A.srcs, A.outs, direct_outs=A.douts)
    pb = R.plan_device(Bs.srcs, Bs.outs, direct_outs=Bs.douts)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(63)
    try:
        for run in range(4):
            A.fill(gen, len(cands), 3, min(c.N for c in cands))
            _copy_inputs(Bs, A)
            pa.run()
            pb.run()
            for x, y in zip(A.outs + A.douts, Bs.outs + Bs.douts):
                assert torch.isfinite(x).all() and torch.equal(x, y), run
        torch.cuda.synchronize()
        R.check_device_errors()
    finally:
        for p in (pa, pb, ga, gb, fpool, ipool):
            p.close()


# ------------------------------------------------------------------------------------------ 4 and 5. tables, bytes
@pytest.mark.parametrize("resident", ["device", "host"])
def test_level_tables_and_bytes(resident):
    render, R = _R()
    rng = np.random.default_rng(641)
    lengths = [1, 63, 64, 65, 4096 * 5 + 3, 60 * RATE]
    ks = [gappy_i16(rng, n) if n > RATE else rng.integers(-32768, 32768, n).astype(np.int16) for n in lengths]
    ks[-1][:5] = -32768
    fl = R.dry_pool([torch.from_numpy(values(k)).cuda() for k in ks], levels=True)
    ip = R.dry_pool(ks, levels=True, host=resident == "host", dtype="int16")
    plain = R.dry_pool(ks, host=resident == "host", dtype="int16")
    try:
        assert fl.level_stride == 1 and ip.level_stride == 64 and plain.level_stride == 64
        for i, k in enumerate(ks):
            full = fl.level_table(i)
            assert torch.equal(ip.level_table(i), full), i
            # the sparse table itself: every 64th entry and the last
            N = len(k)
            m = -(-N // 64) + 1
            q = ip._read(R.lib.ss_dry_pool_level_table(ip._h, i), m, "<f8", ctypes.c_double)
            f = full.cpu().numpy()
            assert np.array_equal(q, f[np.minimum(np.arange(m) * 64, N)]), i
            sig = ip._read(R.lib.ss_dry_pool_signal_i16(ip._h, i), N, "<i2", ctypes.c_int16)
            assert np.array_equal(sig, k), i
        assert plain.level_table(0) is None
        n = len(ks)
        arena = sum(-(-2 * len(k) // 64) * 64 for k in ks)
        tables = 8 * sum(-(-len(k) // 64) + 1 for k in ks)
        if resident == "device":
            assert ip.nbytes == 8 * n + arena + 8 * n + tables and ip.host_nbytes == 0
            assert plain.nbytes == 8 * n + arena and plain.host_nbytes == 0
        else:
            assert ip.nbytes == 8 * n + 8 * n and ip.host_nbytes == arena + tables
            assert plain.nbytes == 8 * n and plain.host_nbytes == arena
        assert fl.nbytes == 8 * n + 8 * sum(len(k) + 1 for k in ks) + 8 * n
    finally:
        for p in (fl, ip, plain):
            p.close()


# ------------------------------------------------------------------------------------------------ 6. clamped picks
@pytest.mark.parametrize("src_resident", ["device", "host"])
def test_clamped_dry_picks_report_bit_4(world, src_resident):
    render, R = _R()
    cands, taps, pools = world["mixedK"]
    ks = i16_signals(651, 3, max(c.N for c in cands))
    fpool, ipool = twin_pools(R, ks, src_resident, "device")
    pool = pools[src_resident]
    A, Bs = DrySlots(pool, fpool, cands, 5000, taps), DrySlots(pool, ipool, cands, 5000, taps)
    pa = R.plan_device(A.srcs, A.outs, direct_outs=A.douts)
    pb = R.plan_device(Bs.srcs, Bs.outs, direct_outs=Bs.douts)
    try:
        torch.cuda.synchronize()
        R.check_device_errors()
        A.picks.copy_(torch.tensor([0, 1, 2, 3], dtype=torch.int32))
        A.dpicks.copy_(torch.tensor([0, 3, -1, 1 << 30], dtype=torch.int32))
        A.starts.copy_(torch.tensor([0, 100, 2000, 7], dtype=torch.int32))
        _copy_inputs(Bs, A)
        for o in A.outs:
            o.fill_(NAN)
        pb.run()
        torch.cuda.synchronize()
        with pytest.raises(IndexError):
            R.check_device_errors()
        R.check_device_errors()                           # cleared
        pa.run()
        torch.cuda.synchronize()
        with pytest.raises(IndexError):
            R.check_device_errors()
        for x, y in zip(A.outs, Bs.outs):
            assert torch.isfinite(x).all() and torch.equal(x, y)
    finally:
        for p in (pa, pb, fpool, ipool):
            p.close()


# ------------------------------------------------------------------------------------------------------ 7. refusals
def test_python_refusals(world):
    render, R = _R()
    good = np.zeros(100, np.int16)
    for bad, match in [([np.full(10, 0.3, np.float32)], "signal 0 has sample 0"),
                       ([good, np.array([0.0, 1.0], np.float32)], "signal 1 has sample 1"),
                       ([torch.full((5,), 1.0 / 65536, device="cuda")], "signal 0 has sample 0"),
                       ([np.ones(10, np.int32)], "int16 or float"),
                       ([torch.ones(10, dtype=torch.int32, device="cuda")], "int16 or float"),
                       ([np.zeros((1 << 23) + 1, np.int16)], "2\\^23"),
                       ([np.zeros((2, 5), np.int16)], "1-D")]:
        with pytest.raises(ValueError, match=match):
            R.dry_pool(bad, dtype="int16")
    with pytest.raises(ValueError, match="dtype"):
        R.dry_pool([good], dtype="float16")
    # a 16-bit pool without tables cannot serve a draw speaker; a device 16-bit pool serves a host pool's slots
    cands, taps, pools = world["aligned"]
    ip = R.dry_pool(i16_signals(661, 2, max(c.N for c in cands)), dtype="int16")
    fdev = R.dry_pool([torch.from_numpy(values(k)).cuda() for k in i16_signals(661, 2, max(c.N for c in cands))])
    try:
        sl = DrySlots(pools["host"], ip, cands, 4000, taps, k=2)
        R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts).close()
        sl = DrySlots(pools["host"], fdev, cands, 4000, taps, k=2)
        with pytest.raises(ValueError, match="host pool"):
            R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
        sl = DrySlots(pools["device"], ip, cands, 4000, taps, k=2)
        st = torch.zeros(1, dtype=torch.int32, device="cuda")
        srcs = [s._replace(window=(st, 4000)) for s in sl.srcs]
        draw = render.CropDraw(st, [0, 1], torch.rand(5, dtype=torch.float64, device="cuda"))
        with pytest.raises(ValueError, match="level tables"):
            R.plan_device(srcs, sl.outs, direct_outs=sl.douts, draws=[draw])
    finally:
        ip.close()
        fdev.close()


def test_c_refusals():
    from sonicsim_b200 import _lib as L
    _, R = _R()
    lib = R.lib
    k = torch.zeros(64, dtype=torch.int16, device="cuda")
    ok = (ctypes.c_void_p * 2)(k.data_ptr(), k.data_ptr())
    odd = (ctypes.c_void_p * 2)(k.data_ptr(), k.data_ptr() + 1)
    null = (ctypes.c_void_p * 2)(k.data_ptr(), None)

    def create(x, lengths, n, flags=0):
        h = ctypes.c_void_p(12345)
        ln = np.asarray(lengths, np.int32)
        st = lib.ss_dry_pool_create_i16(R.ctx, x, ln.ctypes.data if ln.size else None, n, flags, ctypes.byref(h))
        return st, h.value

    st, h = create(ok, [64, 64], 2)
    assert st == L.SS_OK and h
    lib.ss_dry_pool_destroy(ctypes.c_void_p(h))
    for args, want in [((None, [64, 64], 2), L.SS_ERR_INVALID), ((ok, [], 2), L.SS_ERR_INVALID),
                       ((ok, [64, 64], 0), L.SS_ERR_INVALID), ((ok, [64, 64], (1 << 24) + 1), L.SS_ERR_INVALID),
                       ((odd, [64, 64], 2), L.SS_ERR_INVALID), ((null, [64, 64], 2), L.SS_ERR_INVALID),
                       ((ok, [64, 64], 2, 2), L.SS_ERR_INVALID), ((ok, [64, 0], 2), L.SS_ERR_UNSUPPORTED),
                       ((ok, [64, (1 << 23) + 1], 2), L.SS_ERR_UNSUPPORTED),
                       ((ok, [64, -5], 2, L.SS_DRY_LEVELS), L.SS_ERR_UNSUPPORTED)]:
        st, h = create(*args)
        assert st == want, args
        assert h in (None, 0, 12345), args                  # no pool created
    assert lib.ss_dry_pool_level_stride(None) == 0 and lib.ss_dry_pool_signal_i16(None, 0) is None
    fp = R.dry_pool([torch.zeros(64, device="cuda")])
    try:
        assert lib.ss_dry_pool_signal_i16(fp._h, 0) is None and lib.ss_dry_pool_level_stride(fp._h) == 1
    finally:
        fp.close()
