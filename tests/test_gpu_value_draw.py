"""Value draws (render.ValueDraw; ss_plan_create_values) through the real kernels.  Plan A draws its per-run inputs
itself (k_values); plan B is the same plan without value draws, reading the same input tensors, run after A.  Checked:
  1. after every run the drawn tensors equal the CPU emulation (tests/emu/ss_emu_values.cu) for that run's (seed, t);
     the same t draws them again, t + 1 draws others;
  2. bit identity of A and B: stems, direct stems, mixtures, speakers_out, dereverberation targets, rms_db, drawn
     starts and `used`, StemLoudness results and drawn layouts (A's equal B's, which has no value draws), over device,
     host and tap-form host source pools with stream, bed and dry-picked slots; plain start windows in multi-chunk
     plans; one run of A on a side stream behind queued work;
  3. A launches exactly one kernel per run more than B, and check_device_errors stays clean;
  4. refusals: ValueErrors before any C call, and the C ABI's, with *out untouched;
  5. scale: B = 4096 rows, five draws including a u of 101 doubles per row, against the emulation."""
import ctypes

import numpy as np
import pytest
import torch

import value_reference as vr
from gpu_plumbing import _R
from oracle import sonicsim_oracle as so
from pool_worlds import Cand, _host_pool, noises, speakers
from value_reference import Spec

pytestmark = pytest.mark.gpu

TAPS = 40
RATE = 1600
M = 12
WL = 8000
NAN = float("nan")
SLEEP = int(5e8)
SMALL = 1 << 20              # a chunk budget of about one source per chunk
DEFAULT_CHUNK_BYTES = 32 << 20


def signals(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        v = rng.standard_normal(int(rng.integers(lo, hi + 1)))
        v *= rng.uniform(0.05, 0.9) / np.abs(v).max()
        out.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
    return out


def equal_n(seed, n, N=40000):
    rng = np.random.default_rng(seed)
    return [Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 3 + j % 3, 2, 4096),
                 np.round(np.linspace(0, N, 3 + j % 3)).astype(np.int32), TAPS) for j in range(n)]


def static_equal_n(seed, n, N=40000):
    rng = np.random.default_rng(seed)
    return [Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 4096)[0], None) for _ in range(n)]


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    spk, noi = speakers(2101, n=6, taps=TAPS), noises(2102, n=2)
    tap_banks = [R.rir_bank(c.h, False, TAPS, host=True, form="taps") for c in spk]
    pools = {"device": R.source_pool([c.src for c in spk]), "host": _host_pool(R, render, spk, TAPS),
             "taps": R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(spk, tap_banks)]),
             "equal": R.source_pool([c.src for c in equal_n(2103, 6)])}
    npools = {"device": R.source_pool([c.src for c in noi]), "host": _host_pool(R, render, noi),
              "equal": R.source_pool([c.src for c in static_equal_n(2104, 2)])}
    utts = signals(2105, 40, int(0.2 * RATE), int(1.5 * RATE))
    upool = R.dry_pool(utts, levels=True, dtype="int16")
    cpool = R.dry_pool(signals(2106, 9, int(0.3 * RATE), int(4 * RATE)), dtype="int16")
    dpool = R.dry_pool(signals(2107, 5, 52000, 60000), levels=True, dtype="int16")
    yield pools, npools, upool, cpool, dpool
    for p in list(pools.values()) + list(npools.values()) + [upool, cpool, dpool]:
        p.close()
    for b in tap_banks:
        b.close()


def inputs(B, lufs, seed=20261018):
    d = "cuda"
    return dict(scene=torch.zeros(B, dtype=torch.int32, device=d),
                picks=torch.zeros((B, 3), dtype=torch.int32, device=d),
                dpk=torch.zeros(B, dtype=torch.int32, device=d), u=torch.zeros((B, 37), dtype=torch.float64, device=d),
                sirs=torch.zeros((B, 2), device=d), snr=torch.zeros(B, device=d),
                tgs=torch.zeros((B, 2), dtype=torch.float64, device=d),
                tgn=torch.zeros((B, 1), dtype=torch.float64, device=d),
                rng=torch.tensor([seed, 0], dtype=torch.int64, device=d))


def value_list(render, sh, lufs, n_dry):
    """The ValueDraws of a training step over sh, and their Specs for the emulation."""
    r = sh["rng"]
    v = [render.ValueDraw(sh["scene"], r, 0, 2),
         render.ValueDraw(sh["picks"], r, 0, 3, distinct=True, base=sh["scene"], stride=3),
         render.ValueDraw(sh["dpk"], r, 0, n_dry), render.ValueDraw(sh["u"], r),
         render.ValueDraw(sh["sirs"], r, -6, 6), render.ValueDraw(sh["snr"], r, 10, 20)]
    s = [Spec(np.int32, 1, 0, 2), Spec(np.int32, 3, 0, 3, distinct=True, base=0, stride=3),
         Spec(np.int32, 1, 0, n_dry), Spec(np.float64, 37), Spec(np.float32, 2, -6, 6), Spec(np.float32, 1, 10, 20)]
    if lufs:
        v += [render.ValueDraw(sh["tgs"], r, -19, -15), render.ValueDraw(sh["tgn"], r, -26, -22)]
        s += [Spec(np.float64, 2, -19, -15), Spec(np.float64, 1, -26, -22)]
    return v, s


class Step:
    """B examples of a separation step over scene-major pools: two stream speakers and a dry-picked speaker (direct
    stems), a bed noise of the scene, a CropDraw over the speakers that the bed also reads, a mixture with noise_delay
    and dereverberation targets, drawn layouts; `lufs` gives the stream and bed slots a StemLoudness with a result.
    `values`: the plan draws the inputs of `sh` itself."""

    def __init__(self, R, render, pool, npool, upool, cpool, dpool, sh, values, lufs):
        d = "cuda"
        B = sh["scene"].shape[0]
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.used = torch.zeros(B, dtype=torch.int32, device=d)
        self.lay = torch.full((B, 3, 4, M), -1, dtype=torch.int32, device=d)
        self.res = torch.zeros((B, 3, 2), dtype=torch.float64, device=d)
        C = pool.C
        self.outs = [torch.empty((C, WL), device=d) for _ in range(4 * B)]
        self.douts = [torch.empty((C, WL), device=d) if j % 4 < 3 else None for j in range(4 * B)]
        self.mix = torch.empty((B, C, WL), device=d)
        self.spo = torch.empty((B, 3, C, WL), device=d)
        self.tgt = torch.empty((B, 3, C, WL), device=d)
        self.rms = torch.empty((B, 3), device=d)
        totals = [min(pool._sizes) + 3 * RATE, min(pool._sizes), 2 * min(npool._sizes)]
        srcs, draws, mixes, layouts = [], [], [], []
        for b in range(B):
            w = (self.starts[b], WL)
            q = [render.StemLoudness(sh["tgs"][b, k:k + 1] if k < 2 else sh["tgn"][b], self.res[b, k]) if lufs
                 else None for k in range(3)]
            for k in range(2):
                srcs.append(render.Pooled(pool, sh["picks"][b, k], w, TAPS,
                                          render.DryStream(upool, self.lay[b, k, 0], self.lay[b, k, 1], lufs=q[k])))
            srcs.append(render.Pooled(pool, sh["picks"][b, 2], w, TAPS, render.DryPick(dpool, sh["dpk"][b])))
            srcs.append(render.Pooled(npool, sh["scene"][b:b + 1], w, 0,
                                      render.BackgroundStream(cpool, *[self.lay[b, 2, r] for r in range(4)],
                                                              lufs=q[2])))
            draws.append(render.CropDraw(self.starts[b], [4 * b, 4 * b + 1, 4 * b + 2], sh["u"][b], self.used[b],
                                         -35.0))
            mixes.append(render.Mixture([4 * b, 4 * b + 1, 4 * b + 2], [4 * b + 3], sh["sirs"][b], sh["snr"][b],
                                        self.mix[b], self.spo[b], self.rms[b], noise_delay=777, direct_out=self.tgt[b]))
            for k, slot in enumerate((4 * b, 4 * b + 1, 4 * b + 3)):
                layouts.append(render.LayoutDraw(slot, sh["rng"], totals[k], RATE))
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts, mixtures=mixes, draws=draws,
                                  layouts=layouts, values=values)

    def clear(self):
        for t in self.outs + [x for x in self.douts if x is not None] + [self.mix, self.spo, self.tgt, self.rms,
                                                                       self.res]:
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)
        self.lay.fill_(-3)

    def outputs(self):
        return [*self.outs, *[x for x in self.douts if x is not None], self.mix, self.spo, self.tgt, self.rms,
                self.starts, self.used, self.res, self.lay]


def same_bits(a, b):
    if a.dtype in (torch.float32, torch.int32):
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a.view(torch.int64), b.view(torch.int64))


def check_values(sh, specs, names):
    """The drawn tensors sh[names] equal the emulation's values at (seed, t) = sh["rng"]; returns them."""
    rng = sh["rng"].cpu().numpy()
    B = sh[names[0]].shape[0]
    want = vr.emu_rows(vr.load_emu(), specs, B, int(rng[0]), int(rng[1]))
    got = [sh[k].cpu().numpy().reshape(B, -1) for k in names]
    for k, g, w in zip(names, got, want):
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8)), k
    return got


NAMES = ["scene", "picks", "dpk", "u", "sirs", "snr", "tgs", "tgn"]


@pytest.mark.parametrize("src,lufs", [("device", False), ("host", False), ("taps", False), ("equal", True)])
def test_drawn_values_equal_the_emulation_and_render_as_refreshed_ones(world, src, lufs):
    render, R = _R()
    pools, npools, upool, cpool, dpool = world
    npool = npools["equal" if src == "equal" else "host" if src == "host" else "device"]
    B = 2
    sh = inputs(B, lufs)
    values, specs = value_list(render, sh, lufs, dpool.n)
    A = Step(R, render, pools[src], npool, upool, cpool, dpool, sh, values, lufs)
    Z = Step(R, render, pools[src], npool, upool, cpool, dpool, sh, None, lufs)
    side = torch.cuda.Stream()
    names = NAMES[:len(specs)]
    try:
        previous = None
        for run, t in enumerate([3, 3, 4, 900]):
            sh["rng"][1] = t
            for k in names:
                sh[k].fill_(-1)
            A.clear()
            Z.clear()
            torch.cuda.synchronize()
            R.reset_stats()
            if run == 3:                                       # on a side stream behind queued work
                with torch.cuda.stream(side):
                    torch.cuda._sleep(SLEEP)
                    A.plan.run()
                side.synchronize()
            else:
                A.plan.run()
            torch.cuda.synchronize()
            a_launches = R.launch_count()
            R.check_device_errors()
            got = check_values(sh, specs, names)               # 1. the emulation's values for (seed, t)
            if run == 1:
                assert all(np.array_equal(a, b) for a, b in zip(got, previous))
            if run == 2:
                assert not any(np.array_equal(a, b) for a, b in zip(got[3:], previous[3:]))
            previous = got
            R.reset_stats()
            Z.plan.run()
            torch.cuda.synchronize()
            assert a_launches == R.launch_count() + 1          # 3. one launch more
            R.check_device_errors()
            for x, y in zip(A.outputs(), Z.outputs()):         # 2. bit identity, drawn layouts included
                assert same_bits(x, y), run
            assert torch.isfinite(A.mix).all() and (A.used >= 0).all() and (A.lay[:, :, 0, 0] >= 0).any()
            if lufs:
                assert torch.isfinite(A.res[..., 1]).all()
        assert A.plan.is_graph() and Z.plan.is_graph()
    finally:
        A.plan.close()
        Z.plan.close()


@pytest.mark.parametrize("src", ["device", "host", "taps"])
def test_plain_starts_and_picks_in_multi_chunk_plans(world, src):
    """Plain randint windows (no CropDraw) and picks drawn by the plan, over plans of many chunks."""
    render, R = _R()
    pools, npools, upool, cpool, dpool = world
    pool = pools[src]
    B, d = 6, "cuda"
    n_min = min(pool._sizes)
    rng = torch.tensor([-5, 0], dtype=torch.int64, device=d)
    picks = torch.zeros((B, 2), dtype=torch.int32, device=d)
    starts = torch.zeros(B, dtype=torch.int32, device=d)
    dpk = torch.zeros((B, 2), dtype=torch.int32, device=d)
    values = [render.ValueDraw(picks, rng, 0, pool.n, distinct=True), render.ValueDraw(starts, rng, 0, n_min - WL + 1),
              render.ValueDraw(dpk, rng, 0, dpool.n)]
    specs = [Spec(np.int32, 2, 0, pool.n, distinct=True), Spec(np.int32, 1, 0, n_min - WL + 1),
             Spec(np.int32, 2, 0, dpool.n)]
    outs = [[torch.empty((pool.C, WL), device=d) for _ in range(2 * B)] for _ in range(2)]
    douts = [[torch.empty((pool.C, WL), device=d) for _ in range(2 * B)] for _ in range(2)]
    R.set_chunk_bytes(SMALL)
    plans = []
    try:
        for arm in range(2):
            srcs = [render.Pooled(pool, picks[b, k], (starts[b], WL), TAPS, render.DryPick(dpool, dpk[b, k]) if k
                                  else None) for b in range(B) for k in range(2)]
            plans.append(R.plan_device(srcs, outs[arm], direct_outs=douts[arm], values=values if arm == 0 else None))
        for t in (0, 1, 2):
            rng[1] = t
            R.reset_stats()
            plans[0].run()
            torch.cuda.synchronize()
            a = R.launch_count()
            R.check_device_errors()
            check_values(dict(picks=picks, starts=starts, dpk=dpk, rng=rng), specs,
                         ["picks", "starts", "dpk"])
            R.reset_stats()
            plans[1].run()
            torch.cuda.synchronize()
            assert a == R.launch_count() + 1 and a > 8         # many chunks
            R.check_device_errors()
            for x, y in zip(outs[0] + douts[0], outs[1] + douts[1]):
                assert same_bits(x, y), t
    finally:
        R.set_chunk_bytes(DEFAULT_CHUNK_BYTES)
        for p in plans:
            p.close()


# ----------------------------------------------------------------------------------------------------- refusals
class _NoCreate:
    """A library proxy that fails the test if a plan reaches plan creation."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        if name.startswith("ss_plan_create"):
            raise AssertionError("a refused plan reached the C ABI")
        return getattr(self._lib, name)


def small_plan(render, pools, npools, upool, dpool):
    d = "cuda"
    sh = dict(pick=torch.zeros(3, dtype=torch.int32, device=d), dpk=torch.zeros(1, dtype=torch.int32, device=d),
              start=torch.zeros(2, dtype=torch.int32, device=d), u=torch.zeros((1, 8), dtype=torch.float64, device=d),
              sirs=torch.zeros(1, device=d), snr=torch.zeros(1, device=d),
              tg=torch.zeros(1, dtype=torch.float64, device=d), rng=torch.zeros(4, dtype=torch.int64, device=d),
              lay=torch.full((2, M), -1, dtype=torch.int32, device=d), used=torch.zeros(1, dtype=torch.int32, device=d))
    outs = [torch.empty((2, WL), device=d) for _ in range(3)]
    mixo = torch.empty((2, WL), device=d)
    srcs = [render.Pooled(pools["device"], sh["pick"][0:1], (sh["start"][0], WL), 0,
                          render.DryStream(upool, sh["lay"][0], sh["lay"][1])),
            render.Pooled(pools["device"], sh["pick"][1:2], (sh["start"][0], WL), 0, render.DryPick(dpool, sh["dpk"])),
            render.Pooled(npools["device"], sh["pick"][2:3], (sh["start"][1], WL), 0)]
    kw = dict(mixtures=[render.Mixture([0, 1], [2], sh["sirs"], sh["snr"], mixo)],
              draws=[render.CropDraw(sh["start"][0], [0], sh["u"][0], sh["used"])],
              layouts=[render.LayoutDraw(0, sh["rng"][:2], 48000, RATE)])
    return sh, srcs, outs, mixo, kw


def test_python_refusals(world):
    render, R = _R()
    pools, npools, upool, cpool, dpool = world
    sh, srcs, outs, mixo, kw = small_plan(render, pools, npools, upool, dpool)
    d = "cuda"
    r = sh["rng"][2:]
    V = render.ValueDraw
    f = torch.zeros((4, 3), device=d)
    i = torch.zeros(4, dtype=torch.int32, device=d)
    i2 = torch.zeros((4, 2), dtype=torch.int32, device=d)
    big = torch.zeros((1, 4097), dtype=torch.float64, device=d)
    ok = [V(sh["pick"], r, 0, 3), V(sh["dpk"], r, 0, 5, base=sh["pick"][:1], stride=1)]   # (different B: refused)
    cases = [
        [("out", r)], [V(f.cpu(), r)], [V(f, r.cpu())], [V(f, sh["rng"])], [V(f, r.to(torch.int32))],
        [V(f[:, :2], r)], [V(torch.zeros(4, dtype=torch.int64, device=d), r)], [V(big, r)],
        [V(torch.zeros((65536,), device=d), r)], [V(torch.zeros((4, 2, 2), device=d), r)],
        [V(f, torch.zeros(3, dtype=torch.int64, device=d))],
        [V(f, r, 1, 1)], [V(f, r, 2, 1)], [V(f, r, 0, float("inf"))], [V(f, r, float("nan"), 1)],
        [V(f, r, 0, 0.1)],                                                                   # 0.1: not a float32
        [V(f, r, distinct=True)], [V(f, r, base=i)], [V(i, r, 0, 1.5)], [V(i, r, 0, 1 << 31)],
        [V(i, r, -(1 << 31) - 1, 0)], [V(i2, r, 0, 1, distinct=True)],
        [V(torch.zeros((4, 65), dtype=torch.int32, device=d), r, 0, 100, distinct=True)],
        [V(i, r, 0, 3), V(i2, r, 0, 3, base=i)],                                             # no stride
        [V(i, r, 0, 3), V(i2, r, 0, 3, base=i2, stride=1)],                                  # base not earlier
        [V(i2, r, 0, 3), V(i, r, 0, 3, base=i2, stride=1)],                                  # base k = 2
        [V(f[:, 0].contiguous(), r), V(i, r, 0, 3, base=f[:, 0], stride=1)],
        [V(i, r, 0, 3, stride=2)],                                                           # stride, no base
        [V(i, r, 0, 1 << 20), V(i2, r, 0, 3000, base=i, stride=3000)],                       # may overflow
        [V(i, r, 0, 3), V(torch.zeros(5, dtype=torch.int32, device=d), r, 0, 3)],            # rows differ
        ok,
    ]
    meet = [
        [V(sh["lay"][0], r, 0, 3)],                       # a drawn layout
        [V(outs[0].view(-1)[:8].view(torch.int32), r, 0, 3)],   # an output
        [V(mixo.view(-1)[:4], r)],                        # a mixture's output
        [V(sh["start"][0:1], r, 0, 3)],                   # a start a CropDraw writes
        [V(sh["used"], r, 0, 3)],                         # `used`
        [V(sh["rng"][:2].view(torch.int32), r, 0, 3)],    # a layout draw's rng
        [V(r.view(torch.float64), r)],                    # its own rng
        [V(sh["pick"][:2], r, 0, 3), V(sh["pick"][1:], r, 0, 3)],   # another value out
        [V(sh["u"].view(-1)[:4], sh["lay"][0, :4].view(torch.int64))],                # rng over a drawn layout
        [V(sh["u"].view(-1)[:4], outs[1].view(-1)[:4].view(torch.int64))],           # rng over an output
    ]
    lib = R.lib
    R.lib = _NoCreate(lib)
    try:
        for c in cases:
            with pytest.raises(ValueError):
                R.plan_device(srcs, outs, values=c, **kw)
        for c in meet:
            with pytest.raises(ValueError, match="meets"):
                R.plan_device(srcs, outs, values=c, **kw)
    finally:
        R.lib = lib
    # every allowed per-run input may be drawn: picks, dry picks, an undrawn start, sirs, snr, u; targets elsewhere
    allowed = [V(sh["pick"], r, 0, 2), V(sh["dpk"], r, 0, dpool.n), V(sh["start"][1:], r, 0, 100),
               V(sh["sirs"], r, -6, 6), V(sh["snr"], r, 10, 20), V(sh["u"][0], r)]
    for a in allowed:
        R.plan_device(srcs, outs, values=[V(a.out.view(1, -1), a.rng, a.low, a.high)], **kw).close()
    R.plan_device(srcs, outs, values=[V(sh["snr"], r, 10, 20), V(sh["sirs"], r, -6, 6)], **kw).close()


def test_c_abi_refusals(world):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    pools, npools, upool, cpool, dpool = world
    sh, srcs, outs, mixo, kw = small_plan(render, pools, npools, upool, dpool)
    d = "cuda"
    # the plan's own arrays, as plan_device builds them, without render.ValueDraw's checks
    mixtures, draws, layouts = kw["mixtures"], kw["draws"], kw["layouts"]
    dry, streams, bgs = R._device_dry(srcs), R._device_streams(srcs), R._device_bgs(srcs)
    items, n, keep = R._device_items(srcs, outs)
    targets = []
    mixes = R._device_mixes(mixtures, outs, keep, items, targets)
    drw = R._device_draws(draws, srcs, keep)
    lufs = R._device_lufs(srcs, (outs, None, mixtures, draws), keep)
    lay = R._device_layouts(layouts, srcs, (outs, None, mixtures, draws), keep)
    pair = R._device_pair_gains(srcs)
    o = torch.zeros((4, 256), dtype=torch.float64, device=d)      # 8 KB: room for several entries' outs
    rng = torch.zeros(2, dtype=torch.int64, device=d)

    def E(out=None, kind=L.SS_VALUE_F64, rows=4, k=64, base=-1, low=0.0, high=1.0, ilow=0, ihigh=3, stride=0,
          r=None):
        return L.SsValueDraw(out=o.data_ptr() if out is None else out, rng_dev=rng.data_ptr() if r is None else r,
                             kind=kind, rows=rows, k=k, base=base, low=low, high=high, ilow=ilow, ihigh=ihigh,
                             stride=stride)

    def create(entries, count=None, arr=None):
        if arr is None:
            arr = (L.SsValueDraw * len(entries))(*entries) if entries else None
        h = ctypes.c_void_p(12345)
        s = R.lib.ss_plan_create_values(R.ctx, items, n, mixes, 1, drw, 1, dry, pair, 1, None, 0, streams, 1, None, 0,
                                        None, 0, lay, 1, arr, len(entries) if count is None else count,
                                        ctypes.byref(h))
        if s == L.SS_OK:
            R.lib.ss_plan_destroy(h)
            return s
        assert h.value == 12345                                    # *out untouched
        return s

    Int, F32, p0 = L.SS_VALUE_INT, L.SS_VALUE_F32, o.data_ptr()
    one = dict(rows=1, k=1)
    assert create([E()]) == L.SS_OK
    assert create([]) == L.SS_OK                                   # ss_plan_create_layout
    assert create([E(kind=Int, k=1), E(p0 + 64, Int, k=3, base=0, stride=3, ihigh=3),
                   E(p0 + 256, L.SS_VALUE_DISTINCT, k=64, ihigh=64), E(p0 + 2048, F32, k=2, low=-6, high=6)]) == L.SS_OK
    # every per-run input may be drawn: picks, the dry pick, the undrawn start, sirs, snr, u
    assert create([E(sh["pick"].data_ptr(), Int, rows=1, k=3), E(sh["dpk"].data_ptr(), Int, **one),
                   E(sh["start"][1:].data_ptr(), Int, **one), E(sh["sirs"].data_ptr(), F32, low=-6, high=6, **one),
                   E(sh["snr"].data_ptr(), F32, low=10, high=20, **one),
                   E(sh["u"].data_ptr(), rows=1, k=8)]) == L.SS_OK
    invalid = [
        [E(0)], [E(p0 + 4)], [E(r=0)], [E(r=rng.data_ptr() + 4)], [E(kind=4)], [E(kind=-1)],
        [E(rows=0)], [E(rows=65536, k=1)], [E(), E(p0 + 4096, rows=3, k=1)], [E(k=0)], [E(k=4097, rows=1)],
        [E(low=1, high=1)], [E(low=float("nan"))], [E(high=float("inf"))],
        [E(kind=F32, low=0, high=0.1)], [E(kind=Int, k=1), E(p0 + 64, base=0, k=1)],
        [E(kind=Int, ilow=3, ihigh=3)], [E(kind=L.SS_VALUE_DISTINCT, k=65, ihigh=100)],
        [E(kind=L.SS_VALUE_DISTINCT, k=4, ihigh=3)],
        [E(kind=Int, k=1), E(p0 + 64, Int, k=1, base=0, stride=0)],                 # stride < 1
        [E(kind=Int, k=1), E(p0 + 64, Int, k=1, base=1, stride=1)],                 # base not earlier
        [E(kind=Int, k=2), E(p0 + 64, Int, k=1, base=0, stride=1)],                 # base k = 2
        [E(k=1), E(p0 + 64, Int, k=1, base=0, stride=1)],                           # base not int
        [E(kind=Int, k=1, ihigh=1 << 20), E(p0 + 64, Int, k=1, base=0, stride=3000, ihigh=3000)],   # overflow
        [E(), E(p0 + 8)],                                          # outs meet
        [E(r=p0 + 8)],                                             # an out meets an rng
        [E(outs[2].data_ptr(), k=1)],                              # an output
        [E(mixo.data_ptr(), F32, **one)],                          # a mixture's output
        [E(sh["start"].data_ptr(), Int, **one)],                   # the start a CropDraw writes
        [E(sh["used"].data_ptr(), Int, **one)],                    # its `used`
        [E(sh["lay"].data_ptr(), Int, **one)],                     # a drawn layout
        [E(sh["rng"].data_ptr(), Int, **one)],                     # a layout draw's rng
        [E(r=outs[2].data_ptr())],                                 # an rng over an output
        [E(r=sh["lay"].data_ptr())],                               # ... over a drawn layout
        [E(r=sh["used"].data_ptr() - 8)],                          # ... over `used`
    ]
    for b in invalid:
        assert create(b) == L.SS_ERR_INVALID, b
    assert create([E()], count=-1) == L.SS_ERR_INVALID
    many = (L.SsValueDraw * ((1 << 20) + 1))()
    assert create([None] * ((1 << 20) + 1), arr=many) == L.SS_ERR_UNSUPPORTED
    h = ctypes.c_void_p()
    assert R.lib.ss_plan_create_values(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0, None, 0, None, 0,
                                       None, 0, None, 0, None, 1, ctypes.byref(h)) == L.SS_ERR_INVALID and not h.value


# -------------------------------------------------------------------------------------------------------- scale
def test_scale_4096_rows_against_the_emulation():
    render, R = _R()
    B, d = 4096, "cuda"
    rng = torch.tensor([987654321, 11], dtype=torch.int64, device=d)
    scene = torch.zeros(B, dtype=torch.int32, device=d)
    picks = torch.zeros((B, 3), dtype=torch.int32, device=d)
    sirs = torch.zeros((B, 2), device=d)
    snr = torch.zeros(B, device=d)
    u = torch.zeros((B, 101), dtype=torch.float64, device=d)
    values = [render.ValueDraw(scene, rng, 0, 500), render.ValueDraw(picks, rng, 0, 3, True, scene, 3),
              render.ValueDraw(sirs, rng, -6, 6), render.ValueDraw(snr, rng, 10, 20), render.ValueDraw(u, rng)]
    specs = [Spec(np.int32, 1, 0, 500), Spec(np.int32, 3, 0, 3, True, 0, 3), Spec(np.float32, 2, -6, 6),
             Spec(np.float32, 1, 10, 20), Spec(np.float64, 101)]
    c = static_equal_n(2201, 2, N=20000)
    pool = R.source_pool([x.src for x in c])
    out = torch.empty((2, 2000), device=d)
    pick = torch.zeros(1, dtype=torch.int32, device=d)
    plan = R.plan_device([render.Pooled(pool, pick, (0, 2000), 0)], [out], values=values)
    try:
        for t in (11, 12):
            rng[1] = t
            plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            want = vr.emu_rows(vr.load_emu(), specs, B, 987654321, t)
            for g, w in zip((scene, picks, sirs, snr, u), want):
                assert np.array_equal(g.cpu().numpy().reshape(B, -1).view(np.uint8), w.view(np.uint8))
            assert (np.sort(want[1] - 3 * want[0], axis=1) == [0, 1, 2]).all()
            assert 0.49 < want[4].mean() < 0.51
    finally:
        plan.close()
        pool.close()
