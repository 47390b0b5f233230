"""Grouped layout draws (render.LayoutDraw(groups=, group=); ss_plan_create_groups) through the real kernels.
Checked:
  1. the defining property end to end: a plan over a 16-bit pool of G speakers whose stream draws read group g equals,
     bit for bit, the plan over a pool of group g's utterances alone with plain draws at the same (seed, t): stems,
     direct stems, mixtures, speakers_out, rms_db, drawn starts and `used`, StemLoudness results; its layouts are the
     sub-pool's with ids shifted by bounds[g]; over device, host and tap-form source pools and device and host
     utterance pools, one run on a side stream behind queued work;
  2. groups drawn by ValueDraw(distinct=True) in the same plan: distinct speakers per example, every id in its
     speaker's range, rows equal to the CPU emulation (tests/emu/ss_emu_layout_group.cu) at several t, the same t
     gives the same bits twice; the plan's ungrouped stream and bed draws are bit-identical to those of the same plan
     without groups, which launches as many kernels per run;
  3. a clamped group: the run equals group G - 1's (group 0's for -1) and check_device_errors raises IndexError;
  4. refusals: ValueErrors before any C call, and the C ABI's, with *out untouched;
  5. scale: about 1000 speaker groups and 128 grouped rows of m = 128 in one plan."""
import ctypes

import numpy as np
import pytest
import torch

import group_reference as gr
from gpu_plumbing import _R
from oracle import sonicsim_oracle as so
from pool_worlds import Cand, _host_pool, noises, speakers

pytestmark = pytest.mark.gpu

TAPS = 40
RATE = 1600
M = 12
WL = 8000
NAN = float("nan")
SLEEP = int(5e8)
SIZES = [7, 3, 12, 1, 9]                 # utterances per speaker


def signals(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        v = rng.standard_normal(int(rng.integers(lo, hi + 1)))
        v *= rng.uniform(0.05, 0.9) / np.abs(v).max()
        out.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
    return out


def equal_n(seed, n=3, N=40000):
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        b = np.round(np.linspace(0, N, 3 + j)).astype(np.int32)
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 3 + j, 2, 4096), b, TAPS))
    return out


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    spk, noi = speakers(1301, n=3, taps=TAPS), noises(1302, n=3)
    tap_banks = [R.rir_bank(c.h, False, TAPS, host=True, form="taps") for c in spk]
    eq = equal_n(1303)
    pools = {"device": R.source_pool([c.src for c in spk]), "host": _host_pool(R, render, spk, TAPS),
             "taps": R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(spk, tap_banks)]),
             "equal": R.source_pool([c.src for c in eq])}
    npool = R.source_pool([c.src for c in noi])
    utts = signals(1305, sum(SIZES), int(0.2 * RATE), int(1.5 * RATE))
    bounds = np.concatenate([[0], np.cumsum(SIZES)]).astype(np.int32)
    upools = {r: R.dry_pool(utts, levels=True, host=r == "host", dtype="int16") for r in ("device", "host")}
    sub = {(r, g): R.dry_pool(utts[bounds[g]:bounds[g + 1]], levels=True, host=r == "host", dtype="int16")
           for r in ("device", "host") for g in (0, 2, 4)}
    clips = signals(1306, 6, int(0.3 * RATE), int(4 * RATE))
    cpool = R.dry_pool(clips, dtype="int16")
    yield dict(pools=pools, npool=npool, utts=utts, bounds=bounds, upools=upools, sub=sub, clips=clips, cpool=cpool)
    for p in list(pools.values()) + list(upools.values()) + list(sub.values()) + [npool, cpool]:
        p.close()
    for b in tap_banks:
        b.close()


class Step:
    """B examples: two stream speakers (direct stems, a layout draw each, grouped when `bounds` is given, reading
    spk[b, k]), a noise slot (a bed with its own ungrouped draw when `bed`), a CropDraw over the speakers, a mixture;
    `lufs` gives the speakers StemLoudness results.  `values` = G: spk is drawn by ValueDraw(spk, rng, 0, G, distinct)."""

    def __init__(self, R, render, pool, npool, upool, B, bounds, lufs, shared, bed=None, values=None):
        d = "cuda"
        self.B, self.sh = B, shared
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.used = torch.zeros(B, dtype=torch.int32, device=d)
        self.lay = torch.full((B, 3, 4, M), -1, dtype=torch.int32, device=d)
        self.res = torch.zeros((B, 2, 2), dtype=torch.float64, device=d)
        C = pool.C
        self.outs = [torch.empty((C, WL), device=d) for _ in range(3 * B)]
        self.douts = [torch.empty((C, WL), device=d) if j % 3 < 2 else None for j in range(3 * B)]
        self.mix = torch.empty((B, C, WL), device=d)
        self.spo = torch.empty((B, 2, C, WL), device=d)
        self.tgt = torch.empty((B, 2, C, WL), device=d)
        self.rms = torch.empty((B, 2), device=d)
        self.totals = [min(pool._sizes) + 3 * RATE, min(pool._sizes), 2 * min(npool._sizes)]
        sh = shared
        srcs, draws, mixes, layouts = [], [], [], []
        for b in range(B):
            w = (self.starts[b], WL)
            for k in range(2):
                q = render.StemLoudness(sh["targets"][b, k:k + 1], self.res[b, k]) if lufs else None
                srcs.append(render.Pooled(pool, sh["picks"][b, k], w, TAPS,
                                          render.DryStream(upool, self.lay[b, k, 0], self.lay[b, k, 1], lufs=q)))
                gk = dict(groups=bounds, group=sh["spk"][b, k:k + 1]) if bounds is not None else {}
                layouts.append(render.LayoutDraw(3 * b + k, sh["rng"], self.totals[k], RATE, **gk))
            if bed is not None:
                srcs.append(render.Pooled(npool, sh["picks"][b, 2], w, 0,
                                          render.BackgroundStream(bed, *[self.lay[b, 2, r] for r in range(4)])))
                layouts.append(render.LayoutDraw(3 * b + 2, sh["rng"], self.totals[2], RATE))
            else:
                srcs.append(render.Pooled(npool, sh["picks"][b, 2], w, 0))
            draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], sh["u"][b], self.used[b], -35.0))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sh["sirs"][b], sh["snr"][b], self.mix[b],
                                        self.spo[b], self.rms[b], noise_delay=777, direct_out=self.tgt[b]))
        vals = [render.ValueDraw(sh["spk"], sh["rng"], 0, values, distinct=True)] if values else None
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts, mixtures=mixes, draws=draws,
                                  layouts=layouts, values=vals)

    def clear(self):
        for t in self.outs + [x for x in self.douts if x is not None] + [self.mix, self.spo, self.tgt, self.rms,
                                                                       self.res]:
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)
        self.lay.fill_(-5)

    def outputs(self):
        return ([*self.outs, *[x for x in self.douts if x is not None], self.mix, self.spo, self.tgt, self.rms,
                 self.starts, self.used, self.res])


def shared_inputs(B, seed=20261018):
    d = "cuda"
    return dict(picks=torch.zeros((B, 3), dtype=torch.int32, device=d),
                u=torch.zeros((B, 37), dtype=torch.float64, device=d),
                sirs=torch.zeros((B, 1), device=d), snr=torch.zeros(B, device=d),
                targets=torch.zeros((B, 2), dtype=torch.float64, device=d),
                spk=torch.zeros((B, 2), dtype=torch.int32, device=d),
                rng=torch.tensor([seed, 0], dtype=torch.int64, device=d))


def refresh(sh, rng, B, t):
    sh["rng"][1] = t
    sh["picks"].copy_(torch.from_numpy(rng.integers(0, 3, (B, 3)).astype(np.int32)))
    sh["u"].uniform_()
    sh["sirs"].uniform_(-6, 6)
    sh["snr"].uniform_(10, 20)
    sh["targets"].copy_(torch.from_numpy(rng.uniform(-26, -15, (B, 2))))


def same_bits(a, b):
    return torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                       b.view(torch.int32) if b.dtype == torch.float32 else b) or (
        a.dtype == torch.float64 and torch.equal(a.view(torch.int64), b.view(torch.int64)))


def run(R, plan, side=None):
    torch.cuda.synchronize()
    R.reset_stats()
    if side is not None:
        with torch.cuda.stream(side):
            torch.cuda._sleep(SLEEP)
            plan.run()
        side.synchronize()
    else:
        plan.run()
    torch.cuda.synchronize()
    return R.launch_count()


CONFIGS = [("device", "device", 0, False), ("host", "host", 2, False), ("taps", "device", 4, False),
           ("equal", "host", 2, True), ("equal", "device", 0, True)]


@pytest.mark.parametrize("src,ures,g,lufs", CONFIGS)
def test_a_group_of_the_whole_pool_renders_as_its_own_pool(world, src, ures, g, lufs):
    render, R = _R()
    B, bounds = 2, world["bounds"]
    sh = shared_inputs(B)
    sh["spk"].fill_(g)
    A = Step(R, render, world["pools"][src], world["npool"], world["upools"][ures], B, bounds, lufs, sh)
    Z = Step(R, render, world["pools"][src], world["npool"], world["sub"][(ures, g)], B, None, lufs, sh)
    rng = np.random.default_rng(9)
    side = torch.cuda.Stream()
    lo = int(bounds[g])
    try:
        for i, t in enumerate([3, 4, 900]):
            refresh(sh, rng, B, t)
            A.clear()
            Z.clear()
            a_launches = run(R, A.plan, side if i == 2 else None)
            R.check_device_errors()
            z_launches = run(R, Z.plan)
            R.check_device_errors()
            assert a_launches == z_launches
            la, lz = A.lay[:, :2, :2].cpu().numpy(), Z.lay[:, :2, :2].cpu().numpy()
            assert np.array_equal(la[:, :, 0], gr.shifted(lz[:, :, 0], lo)), t
            assert np.array_equal(la[:, :, 1], lz[:, :, 1]), t
            assert (la[:, :, 0] >= 0).any()
            for x, y in zip(A.outputs(), Z.outputs()):
                assert same_bits(x, y), t
            assert torch.isfinite(A.mix).all() and (A.used >= 0).all()
            if lufs:
                assert torch.isfinite(A.res[..., 1]).all()
        assert A.plan.is_graph()
    finally:
        A.plan.close()
        Z.plan.close()


def test_distinct_speakers_drawn_in_the_plan(world):
    render, R = _R()
    B, bounds, G = 3, world["bounds"], len(SIZES)
    lengths = [u.size for u in world["utts"]]
    sh = shared_inputs(B, seed=-5)
    shp = dict(sh, spk=torch.zeros_like(sh["spk"]))
    pool, npool, upool = world["pools"]["device"], world["npool"], world["upools"]["device"]
    A = Step(R, render, pool, npool, upool, B, bounds, False, sh, bed=world["cpool"], values=G)
    P = Step(R, render, pool, npool, upool, B, None, False, shp, bed=world["cpool"], values=G)
    rng = np.random.default_rng(10)
    try:
        previous = None
        for run_i, t in enumerate([1, 1, 2, 77]):
            refresh(sh, rng, B, t)
            A.clear()
            P.clear()
            a_launches = run(R, A.plan)
            R.check_device_errors()
            p_launches = run(R, P.plan)
            R.check_device_errors()
            assert a_launches == p_launches                    # groups launch no kernel more
            spk = sh["spk"].cpu().numpy()
            assert ((spk >= 0) & (spk < G)).all() and (spk[:, 0] != spk[:, 1]).all()
            assert torch.equal(shp["spk"], sh["spk"])          # the same value draw in both plans
            la, lp = A.lay.cpu().numpy(), P.lay.cpu().numpy()
            seed_t = sh["rng"].cpu().numpy()
            for b in range(B):
                for k in range(2):
                    r, g = 3 * b + k, int(spk[b, k])           # layout index: 3 per example
                    ids, offs, err = gr.grouped_rows(seed_t, r, lengths, A.totals[k], M, 10 * RATE, bounds, g)
                    assert err == 0
                    assert np.array_equal(la[b, k, 0], ids[0]) and np.array_equal(la[b, k, 1], offs[0]), (t, b, k)
                    v = la[b, k, 0][la[b, k, 0] >= 0]
                    assert ((v >= bounds[g]) & (v < bounds[g + 1])).all()
                    pids, poffs = gr.plain_rows(seed_t, r, lengths, A.totals[k], M, 10 * RATE)
                    assert np.array_equal(lp[b, k, 0], pids[0]) and np.array_equal(lp[b, k, 1], poffs[0])
                assert np.array_equal(la[b, 2], lp[b, 2])      # the ungrouped bed draw, bit for bit
            assert (la[:, 2, 0] >= 0).any()
            if run_i == 1:                                     # the same (seed, t): the same speakers and layouts
                assert np.array_equal(la, previous[0]) and np.array_equal(spk, previous[1])
            if run_i == 2:
                assert not np.array_equal(la, previous[0])
            previous = (la, spk)
            assert torch.isfinite(A.mix).all()
    finally:
        A.plan.close()
        P.plan.close()


def test_a_clamped_group_is_the_last_group_and_is_reported(world):
    render, R = _R()
    B, bounds, G = 2, world["bounds"], len(SIZES)
    pool, npool, upool = world["pools"]["device"], world["npool"], world["upools"]["device"]
    sh = shared_inputs(B, seed=3)
    A = Step(R, render, pool, npool, upool, B, bounds, False, sh)
    rng = np.random.default_rng(11)
    try:
        refresh(sh, rng, B, 5)
        for bad, good in ((G, G - 1), (-1, 0)):
            sh["spk"].fill_(bad)
            A.clear()
            run(R, A.plan)
            with pytest.raises(IndexError, match="group"):
                R.check_device_errors()
            R.check_device_errors()                            # (the call cleared the bit)
            got = [x.clone() for x in A.outputs()] + [A.lay.clone()]
            sh["spk"].fill_(good)
            A.clear()
            run(R, A.plan)
            R.check_device_errors()
            for x, y in zip(got, A.outputs() + [A.lay]):
                assert same_bits(x, y)
    finally:
        A.plan.close()


# ----------------------------------------------------------------------------------------------------- refusals
class _NoCreate:
    """A library proxy that fails the test if a plan reaches ss_plan_create_groups."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        if name.startswith("ss_plan_create"):
            raise AssertionError("a refused plan reached the C ABI")
        return getattr(self._lib, name)


def test_python_refusals(world):
    render, R = _R()
    d = "cuda"
    bounds = world["bounds"]
    n = int(bounds[-1])
    lay = torch.full((2, 4, M), -1, dtype=torch.int32, device=d)
    pick = torch.zeros(3, dtype=torch.int32, device=d)
    rng = torch.zeros(2, dtype=torch.int64, device=d)
    spk = torch.zeros(4, dtype=torch.int32, device=d)
    outs = [torch.empty((2, WL), device=d) for _ in range(2)]
    srcs = [render.Pooled(world["pools"]["device"], pick[0:1], (0, WL), 0,
                          render.DryStream(world["upools"]["device"], lay[0, 0], lay[0, 1])),
            render.Pooled(world["npool"], pick[1:2], (0, WL), 0,
                          render.BackgroundStream(world["cpool"], *lay[1]))]

    def L(slot=0, groups=bounds, group=spk[:1]):
        return render.LayoutDraw(slot, rng, 48000, RATE, groups=groups, group=group)

    cases = [[L(1, [0, 6])], [L(groups=None)], [L(group=None)], [L(groups=[0, n - 1])], [L(groups=[1, n])],
             [L(groups=[0, 3, 3, n])], [L(groups=[0, 5, 2, n])], [L(group=spk[:1].long())], [L(group=spk[:1].cpu())],
             [L(group=spk[:2])], [L(group=lay[0, 0, :1])],           # a group the plan writes (its own layout)
             [L(group=outs[0].view(-1)[:1].view(torch.int32))]]      # ... an output
    many = R.dry_pool([np.ones(1, np.int16)] * 1100 + [np.ones(5, np.int16)] * 4, dtype="int16")
    big = [srcs[0]._replace(dry=render.DryStream(many, lay[0, 0], lay[0, 1]))] + srcs[1:]
    lib = R.lib
    R.lib = _NoCreate(lib)
    try:
        for c in cases:
            with pytest.raises(ValueError):
                R.plan_device(srcs, outs, layouts=c)
        with pytest.raises(ValueError, match="could select"):
            R.plan_device(big, outs, layouts=[L(groups=[0, 1100, 1104], group=spk[:1])._replace(total=1025)])
    finally:
        R.lib = lib
    # a value draw may write the group; a group of 1100 one-sample utterances reaches K = 1024 exactly
    p = R.plan_device(srcs, outs, layouts=[L(group=spk[:1])],
                      values=[render.ValueDraw(spk[:1], rng, 0, len(SIZES))])
    p.close()
    p = R.plan_device(big, outs, layouts=[L(groups=[0, 1100, 1104], group=spk[:1])._replace(total=1024)])
    p.close()
    many.close()


def test_c_abi_refusals(world):
    from sonicsim_b200 import _lib as Lb
    render, R = _R()
    d = "cuda"
    bounds = world["bounds"]
    lay = torch.full((2, 4, M), -1, dtype=torch.int32, device=d)
    pick = torch.zeros(3, dtype=torch.int32, device=d)
    rng = torch.zeros(2, dtype=torch.int64, device=d)
    spk = torch.zeros(4, dtype=torch.int32, device=d)
    o = [torch.empty((2, WL), device=d) for _ in range(3)]
    srcs = [render.Pooled(world["pools"]["device"], pick[0:1], (0, WL), 0),
            render.Pooled(world["npool"], pick[1:2], (0, WL), 0), render.Pooled(world["npool"], pick[2:3], (0, WL), 0)]
    items, n, keep = R._device_items(srcs, o)
    strm = (Lb.SsDryStream * 1)(Lb.SsDryStream(slot=0, pool=world["upools"]["device"]._h.value,
                                               ids_dev=lay[0, 0].data_ptr(), offsets_dev=lay[0, 1].data_ptr(), m=M))
    bgs = (Lb.SsBgStream * 1)(Lb.SsBgStream(slot=1, pool=world["cpool"]._h.value, ids_dev=lay[1, 0].data_ptr(),
                                            offsets_dev=lay[1, 1].data_ptr(), heads_dev=lay[1, 2].data_ptr(),
                                            counts_dev=lay[1, 3].data_ptr(), m=M))
    lays = (Lb.SsLayoutDraw * 2)(Lb.SsLayoutDraw(slot=0, rng_dev=rng.data_ptr(), total=48000, sample_rate=RATE),
                                 Lb.SsLayoutDraw(slot=1, rng_dev=rng.data_ptr(), total=48000, sample_rate=RATE))
    vals = (Lb.SsValueDraw * 1)(Lb.SsValueDraw(out=spk.data_ptr(), rng_dev=rng.data_ptr(), kind=Lb.SS_VALUE_INT,
                                               rows=1, k=1, base=-1, ilow=0, ihigh=len(SIZES)))
    good = np.ascontiguousarray(bounds, dtype=np.int32)
    holds = []

    def E(layout=0, b=good, g=None, G=None):
        b = np.ascontiguousarray(b, dtype=np.int32)
        holds.append(b)
        return Lb.SsLayoutGroup(layout=layout, n_groups=b.size - 1 if G is None else G, bounds=b.ctypes.data,
                                group_dev=spk.data_ptr() if g is None else g)

    def create(entries, count=None, values=False, arr=None):
        if arr is None:
            arr = (Lb.SsLayoutGroup * len(entries))(*entries) if entries else None
        h = ctypes.c_void_p(12345)
        st = R.lib.ss_plan_create_groups(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0, strm, 1, bgs, 1,
                                         None, 0, lays, 2, vals if values else None, 1 if values else 0, arr,
                                         len(entries) if count is None else count, ctypes.byref(h))
        if st == Lb.SS_OK:
            R.lib.ss_plan_destroy(h)
            return st
        assert h.value == 12345                                    # *out untouched
        return st

    assert create([E()]) == Lb.SS_OK
    assert create([]) == Lb.SS_OK                                  # ss_plan_create_values
    assert create([E()], values=True) == Lb.SS_OK                  # a value draw writes the group
    assert create([E(b=[0, int(bounds[-1])])]) == Lb.SS_OK        # G = 1
    invalid = [[E(-1)], [E(2)], [E(), E()], [E(1, b=[0, 6])], [E(b=[0, 5, 5, int(bounds[-1])])],
               [E(b=[1, int(bounds[-1])])], [E(b=[0, int(bounds[-1]) + 1])], [E(b=[0, 3, 2, int(bounds[-1])])],
               [E(G=0)], [E(g=0)], [E(g=spk.data_ptr() + 2)],
               [E(g=lay[0, 1].data_ptr())],                       # over a layout the plan writes
               [E(g=o[1].data_ptr())]]                            # ... over an output
    for b in invalid:
        assert create(b) == Lb.SS_ERR_INVALID, b
    assert create([E()], count=-1) == Lb.SS_ERR_INVALID
    assert create([E()], count=1, arr=ctypes.POINTER(Lb.SsLayoutGroup)()) == Lb.SS_ERR_INVALID
    e = E()
    e.bounds = None
    assert create([e]) == Lb.SS_ERR_INVALID
    many = R.dry_pool([np.ones(1, np.int16)] * 1100 + [np.ones(5, np.int16)] * 4, dtype="int16")
    strm[0].pool = many._h.value
    lays[0].total = 1024
    assert create([E(b=[0, 1100, 1104])]) == Lb.SS_OK
    lays[0].total = 1025
    assert create([E(b=[0, 1100, 1104])]) == Lb.SS_ERR_UNSUPPORTED
    assert create([E(b=[0, 600, 1104])]) == Lb.SS_OK              # ungrouped it would select 1025
    strm[0].pool = world["upools"]["device"]._h.value
    lays[0].total = 48000
    many.close()


# -------------------------------------------------------------------------------------------------------- scale
def test_a_thousand_speakers_and_128_rows():
    from sonicsim_b200 import dry
    render, R = _R()
    rng = np.random.default_rng(13)
    sizes = rng.integers(1, 40, 1000)
    sizes[17] = 900
    utts = [np.clip(np.round(rng.standard_normal(int(k)) * 8000), -32768, 32767).astype(np.int16)
            for k in rng.integers(25, 65, int(sizes.sum()))]
    lengths = [u.size for u in utts]
    bounds = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    total = 30000
    K = dry.long_audio_max_selected(lengths, total, bounds)
    assert 500 <= K <= 1024
    cands = [Cand(so.synth_dry(np.random.default_rng(s), 20000), so.synth_rirs(np.random.default_rng(s), 1, 2, 4096)[0],
                  None) for s in (1401, 1402)]
    pool = R.source_pool([c.src for c in cands])
    up = R.dry_pool(utts, dtype="int16")
    S, m, wl = 128, 128, 2000
    d = "cuda"
    picks = torch.from_numpy(rng.integers(0, 2, S).astype(np.int32)).to(d)
    group = torch.from_numpy(rng.integers(0, 1000, S).astype(np.int32)).to(d)
    group[:4] = torch.tensor([17, 0, 999, 17], dtype=torch.int32)
    lays = [torch.full((2, S, m), -1, dtype=torch.int32, device=d) for _ in range(2)]
    rng_t = torch.tensor([91, 5], dtype=torch.int64, device=d)
    outs = [[torch.empty((2, wl), device=d) for _ in range(S)] for _ in range(2)]
    starts = rng.integers(0, 20000 - wl, S).tolist()
    plans = []
    try:
        for arm in range(2):
            srcs = [render.Pooled(pool, picks[j:j + 1], (starts[j], wl), 0,
                                  render.DryStream(up, lays[arm][0, j], lays[arm][1, j])) for j in range(S)]
            plans.append(R.plan_device(srcs, outs[arm], layouts=[
                render.LayoutDraw(j, rng_t, total, 1, groups=bounds, group=group[j:j + 1]) for j in range(S)]
                if arm == 0 else None))
        for t in (0, 1):
            rng_t[1] += t
            plans[0].run()
            torch.cuda.synchronize()
            R.check_device_errors()
            got = lays[0].cpu().numpy()
            seed_t, gs = rng_t.cpu().numpy(), group.cpu().numpy()
            for j in list(range(4)) + list(range(4, S, 9)):
                ids, offs, err = gr.grouped_rows(seed_t, j, lengths, total, m, 10, bounds, int(gs[j]))
                assert err == 0 and np.array_equal(got[0, j], ids[0]) and np.array_equal(got[1, j], offs[0]), (t, j)
            assert (got[0, 0] >= 0).sum() == m                 # the 900-utterance speaker reaches the m = 128 cut
            lays[1].copy_(lays[0])
            plans[1].run()
            torch.cuda.synchronize()
            R.check_device_errors()
            for x, y in zip(outs[0], outs[1]):
                assert same_bits(x, y)
    finally:
        for p in plans:
            p.close()
        up.close()
        pool.close()
