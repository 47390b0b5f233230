"""Layout draws (render.LayoutDraw; ss_plan_create_layout) through the real kernels.  Plan A draws its stream and bed
layouts itself (k_layout); plan B is the same plan without draws, whose layout tensors are filled from A's after A's
run.  Checked:
  1. after every run A's layout tensors equal the CPU emulation's rows (tests/emu/ss_emu_layout.cu) for that run's
     (seed, t); the same t draws them again, t + 1 draws others;
  2. bit identity of A and B: stems, direct stems, mixtures, speakers_out, dereverberation targets, rms_db, drawn
     starts and `used`, StemLoudness results, over device, host and tap-form host source pools, device and host 16-bit
     utterance pools, float32 and 16-bit clip pools; one run of each on a side stream behind queued work;
  3. A launches exactly one kernel per run more than B, and check_device_errors stays clean;
  4. refusals: ValueErrors before any C call, and the C ABI's, with *out untouched;
  5. scale: one plan of 300 stream draws over 3000 short utterances, rows cut at m = 128 with K near the cap."""
import ctypes

import numpy as np
import pytest
import torch

from gpu_plumbing import _R
from layout_reference import load_emu
from oracle import sonicsim_oracle as so
from pool_worlds import Cand, _host_pool, noises, speakers

pytestmark = pytest.mark.gpu

TAPS = 40
RATE = 1600                  # gaps and tails of up to 1 s at 1.6 kHz: several utterances per stream
M = 12
WL = 8000
NAN = float("nan")
SLEEP = int(5e8)


def emu_rows(rng_pair, r, lengths, total, m, sr, bed, select=None):
    from sonicsim_b200 import dry
    lib = load_emu()
    L = np.ascontiguousarray(lengths, dtype=np.int32)
    S = None if select is None else np.ascontiguousarray(select, dtype=np.int32)
    K = (dry.background_audio_max_selected(L if S is None else S, total) if bed
         else dry.long_audio_max_selected(L, total))
    rng = np.ascontiguousarray(rng_pair, dtype=np.int64)
    out = [np.zeros(m, np.int32) for _ in range(4)]
    lib.emu_layout_rows(rng.ctypes.data, 1, r, L.ctypes.data, None if S is None else S.ctypes.data, L.size, m, total,
                        10 * sr, K, out[0].ctypes.data, out[1].ctypes.data, out[2].ctypes.data if bed else None,
                        out[3].ctypes.data if bed else None)
    return out if bed else out[:2]


def signals(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    i16, f32 = [], []
    for _ in range(n):
        k = int(rng.integers(lo, hi + 1))
        v = rng.standard_normal(k)
        v *= rng.uniform(0.05, 0.9) / np.abs(v).max()
        i16.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
        f32.append((v + rng.standard_normal(k) * 1e-6).astype(np.float32))
    return {"int16": i16, "float32": f32}


def equal_n(seed, n=3, N=40000):
    """Aligned speakers of one N (loudness slots need it)."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        P = 3 + j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b, TAPS))
    return out


def static_equal_n(seed, n=3, N=40000):
    rng = np.random.default_rng(seed)
    return [Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 4096)[0], None) for _ in range(n)]


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    spk, noi = speakers(1101, n=3, taps=TAPS), noises(1102, n=3)
    tap_banks = [R.rir_bank(c.h, False, TAPS, host=True, form="taps") for c in spk]
    eq, eqn = equal_n(1103), static_equal_n(1104)
    pools = {"device": R.source_pool([c.src for c in spk]), "host": _host_pool(R, render, spk, TAPS),
             "taps": R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(spk, tap_banks)]),
             "equal": R.source_pool([c.src for c in eq])}
    npools = {"device": R.source_pool([c.src for c in noi]), "host": _host_pool(R, render, noi),
              "equal": R.source_pool([c.src for c in eqn])}
    utts = signals(1105, 40, int(0.2 * RATE), int(1.5 * RATE))["int16"]
    upools = {r: R.dry_pool(utts, levels=True, host=r == "host", dtype="int16") for r in ("device", "host")}
    clips = signals(1106, 9, int(0.3 * RATE), int(4 * RATE))
    cpools = {(d, r): R.dry_pool(clips[d] if r == "host" or d == "int16" else [torch.from_numpy(v).cuda()
                                                                               for v in clips[d]],
                                 host=r == "host", dtype=d)
              for d in ("float32", "int16") for r in ("device", "host")}
    yield pools, npools, upools, cpools, utts, clips
    for p in list(pools.values()) + list(npools.values()) + list(upools.values()) + list(cpools.values()):
        p.close()
    for b in tap_banks:
        b.close()


class Step:
    """B examples of a training step: two stream speakers (direct stems) and a bed noise slot, a CropDraw over the
    speakers that the bed also reads, a mixture with noise_delay and dereverberation targets; `lufs` gives every slot
    a StemLoudness with a result.  `shared`: the read-only inputs (picks, u, sirs, snr, targets) of the other arm."""

    def __init__(self, R, render, pool, npool, upool, cpool, B, draw, lufs, shared=None, select=None):
        d = "cuda"
        self.B = B
        if shared is None:
            shared = dict(picks=torch.zeros((B, 3), dtype=torch.int32, device=d),
                          u=torch.zeros((B, 37), dtype=torch.float64, device=d),
                          sirs=torch.zeros((B, 1), device=d), snr=torch.zeros(B, device=d),
                          targets=torch.zeros((B, 3), dtype=torch.float64, device=d),
                          rng=torch.tensor([20261018, 0], dtype=torch.int64, device=d))
        self.shared = shared
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.used = torch.zeros(B, dtype=torch.int32, device=d)
        self.lay = torch.full((B, 3, 4, M), -1, dtype=torch.int32, device=d)
        self.res = torch.zeros((B, 3, 2), dtype=torch.float64, device=d)
        C = pool.C
        self.outs = [torch.empty((C, WL), device=d) for _ in range(3 * B)]
        self.douts = [torch.empty((C, WL), device=d) if j % 3 < 2 else None for j in range(3 * B)]
        self.mix = torch.empty((B, C, WL), device=d)
        self.spo = torch.empty((B, 2, C, WL), device=d)
        self.tgt = torch.empty((B, 2, C, WL), device=d)
        self.rms = torch.empty((B, 2), device=d)
        self.totals = [min(pool._sizes) + 3 * RATE, min(pool._sizes), 2 * min(npool._sizes)]
        srcs, draws, mixes, layouts = [], [], [], []
        sh = shared
        for b in range(B):
            w = (self.starts[b], WL)
            q = [render.StemLoudness(sh["targets"][b, k:k + 1], self.res[b, k]) if lufs else None for k in range(3)]
            for k in range(2):
                srcs.append(render.Pooled(pool, sh["picks"][b, k], w, TAPS,
                                          render.DryStream(upool, self.lay[b, k, 0], self.lay[b, k, 1], lufs=q[k])))
            srcs.append(render.Pooled(npool, sh["picks"][b, 2], w, 0,
                                      render.BackgroundStream(cpool, *[self.lay[b, 2, r] for r in range(4)],
                                                              lufs=q[2])))
            draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], sh["u"][b], self.used[b], -35.0))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sh["sirs"][b], sh["snr"][b], self.mix[b],
                                        self.spo[b], self.rms[b], noise_delay=777, direct_out=self.tgt[b]))
            if draw:
                for k in range(3):
                    layouts.append(render.LayoutDraw(3 * b + k, sh["rng"], self.totals[k], RATE,
                                                     select if k == 2 else None))
        self.layouts = layouts
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts, mixtures=mixes, draws=draws,
                                  layouts=layouts or None)

    def clear(self):
        for t in self.outs + [x for x in self.douts if x is not None] + [self.mix, self.spo, self.tgt, self.rms,
                                                                       self.res]:
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)

    def outputs(self):
        return ([*self.outs, *[x for x in self.douts if x is not None], self.mix, self.spo, self.tgt, self.rms,
                 self.starts, self.used, self.res])


def same_bits(a, b):
    return torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                       b.view(torch.int32) if b.dtype == torch.float32 else b) or (
        a.dtype == torch.float64 and torch.equal(a.view(torch.int64), b.view(torch.int64)))


CONFIGS = [("device", "device", ("float32", "device"), False), ("host", "host", ("int16", "host"), False),
           ("taps", "device", ("float32", "host"), False), ("device", "host", ("int16", "device"), False),
           ("equal", "device", ("int16", "device"), True), ("equal", "host", ("float32", "device"), True)]


@pytest.mark.parametrize("src,ures,clip,lufs", CONFIGS)
def test_drawn_layouts_equal_the_emulation_and_render_as_prefilled_ones(world, src, ures, clip, lufs):
    render, R = _R()
    pools, npools, upools, cpools, utts, clips = world
    npool = npools["equal" if src == "equal" else "device" if src != "host" else "host"]
    cl = clips[clip[0]]
    select = [(c.size * 441) // 160 for c in cl] if clip[0] == "int16" else None
    B = 2
    A = Step(R, render, pools[src], npool, upools[ures], cpools[clip], B, True, lufs, select=select)
    Z = Step(R, render, pools[src], npool, upools[ures], cpools[clip], B, False, lufs, shared=A.shared)
    sh = A.shared
    rng = np.random.default_rng(5)
    side = torch.cuda.Stream()
    ulen, clen = [u.size for u in utts], [c.size for c in cl]
    try:
        previous = None
        for run, t in enumerate([3, 3, 4, 900]):
            sh["rng"][1] = t
            sh["picks"].copy_(torch.from_numpy(rng.integers(0, 3, (B, 3)).astype(np.int32)))
            sh["u"].uniform_()
            sh["sirs"].uniform_(-6, 6)
            sh["snr"].uniform_(10, 20)
            sh["targets"].copy_(torch.from_numpy(rng.uniform(-26, -15, (B, 3))))
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
            lay = A.lay.cpu().numpy()
            for b in range(B):                                 # 1. the emulation's rows for (seed, t)
                for k in range(3):
                    r, bed = 3 * b + k, k == 2
                    want = emu_rows(sh["rng"].cpu().numpy(), r, clen if bed else ulen, A.totals[k], M, RATE, bed,
                                    select if bed else None)
                    for q, v in enumerate(want):
                        assert np.array_equal(lay[b, k, q], v), (run, b, k, q)
            if run == 1:
                assert np.array_equal(lay, previous)           # the same t draws the same layouts
            if run == 2:
                assert not np.array_equal(lay, previous)       # t + 1 others
            previous = lay
            assert (lay[:, :2, 0] >= 0).sum() > B and (lay[:, 2, 0] >= 0).sum() >= B
            Z.lay.copy_(A.lay)
            R.reset_stats()
            Z.plan.run()
            torch.cuda.synchronize()
            assert a_launches == R.launch_count() + 1          # 3. one launch more
            R.check_device_errors()
            for x, y in zip(A.outputs(), Z.outputs()):         # 2. bit identity
                assert same_bits(x, y), run
            assert torch.isfinite(A.mix).all() and (A.used >= 0).all()
            if lufs:
                assert torch.isfinite(A.res[..., 1]).all()
        assert A.plan.is_graph()
    finally:
        A.plan.close()
        Z.plan.close()


# ----------------------------------------------------------------------------------------------------- refusals
class _NoCreate:
    """A library proxy that fails the test if a plan reaches ss_plan_create_layout."""

    def __init__(self, lib):
        self._lib = lib

    def __getattr__(self, name):
        if name == "ss_plan_create_layout":
            raise AssertionError("a refused plan reached the C ABI")
        return getattr(self._lib, name)


def test_python_refusals(world):
    render, R = _R()
    pools, npools, upools, cpools, utts, clips = world
    d = "cuda"
    lay = torch.full((3, 4, M), -1, dtype=torch.int32, device=d)
    pick = torch.zeros(3, dtype=torch.int32, device=d)
    rng = torch.zeros(4, dtype=torch.int64, device=d)
    outs = [torch.empty((2, WL), device=d) for _ in range(4)]
    srcs = [render.Pooled(pools["device"], pick[0:1], (0, WL), 0,
                          render.DryStream(upools["device"], lay[0, 0], lay[0, 1])),
            render.Pooled(npools["device"], pick[1:2], (0, WL), 0,
                          render.BackgroundStream(cpools[("int16", "device")], *lay[1])),
            render.Pooled(npools["device"], pick[2:3], (0, WL), 0),
            render.Pooled(npools["device"], pick[2:3], (0, WL), 0,
                          render.BackgroundStream(cpools[("int16", "device")], *lay[2]))]
    n_clips = len(clips["int16"])
    ok = render.LayoutDraw(0, rng[:2], 48000, RATE)
    cases = [
        [("slot", 0)], [render.LayoutDraw(4, rng[:2], 1000)], [render.LayoutDraw(2, rng[:2], 1000)],
        [ok, render.LayoutDraw(0, rng[2:], 1000)],
        [render.LayoutDraw(0, rng[:2].cpu(), 1000)], [render.LayoutDraw(0, rng, 1000)],
        [render.LayoutDraw(0, rng[:2].to(torch.int32), 1000)],
        [render.LayoutDraw(0, rng[:2], 0)], [render.LayoutDraw(0, rng[:2], 1000, 0)],
        [render.LayoutDraw(0, rng[:2], 1000, select_lengths=[1] * len(utts))],
        [render.LayoutDraw(1, rng[:2], 1000, select_lengths=[1] * (n_clips - 1))],
        [render.LayoutDraw(1, rng[:2], 1000, select_lengths=[-1] + [1] * (n_clips - 1))],
        [render.LayoutDraw(0, lay[0, 0, :4].view(torch.int64)[:2], 1000)],          # rng over a drawn layout
        [render.LayoutDraw(0, outs[0].view(-1)[:4].view(torch.int64), 1000)],        # rng over an output
    ]
    # a drawn layout meeting another tensor: the bed's ids are another slot's offsets, or its pick
    shared = list(srcs)
    shared[3] = srcs[3]._replace(dry=render.BackgroundStream(cpools[("int16", "device")], lay[1, 1], *lay[2][1:]))
    # K above 1024: a stream over 1100 one-sample utterances
    many = R.dry_pool([np.ones(1, np.int16)] * 1100, dtype="int16")
    big = [srcs[0]._replace(dry=render.DryStream(many, lay[0, 0], lay[0, 1]))] + srcs[1:]
    lib = R.lib
    R.lib = _NoCreate(lib)
    try:
        for c in cases:
            with pytest.raises(ValueError):
                R.plan_device(srcs, outs, layouts=c)
        with pytest.raises(ValueError, match="meets"):
            R.plan_device(shared, outs, layouts=[render.LayoutDraw(3, rng[:2], 1000)])
        with pytest.raises(ValueError, match="could select"):
            R.plan_device(big, outs, layouts=[render.LayoutDraw(0, rng[:2], 2000)])
    finally:
        R.lib = lib
    p = R.plan_device(srcs, outs, layouts=[ok, render.LayoutDraw(1, rng[2:], 1000, 16000, [5] * n_clips)])
    p.close()
    p = R.plan_device(big, outs, layouts=[render.LayoutDraw(0, rng[:2], 1024)])   # K = 1024 exactly
    p.close()
    many.close()


def test_c_abi_refusals(world):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    pools, npools, upools, cpools, utts, clips = world
    d = "cuda"
    lay = torch.full((2, 4, M), -1, dtype=torch.int32, device=d)
    pick = torch.zeros(3, dtype=torch.int32, device=d)
    rng = torch.zeros(4, dtype=torch.int64, device=d)
    o = [torch.empty((2, WL), device=d) for _ in range(3)]
    srcs = [render.Pooled(pools["device"], pick[0:1], (0, WL), 0), render.Pooled(npools["device"], pick[1:2], (0, WL), 0),
            render.Pooled(npools["device"], pick[2:3], (0, WL), 0)]
    items, n, keep = R._device_items(srcs, o)
    strm = (L.SsDryStream * 1)(L.SsDryStream(slot=0, pool=upools["device"]._h.value, ids_dev=lay[0, 0].data_ptr(),
                                             offsets_dev=lay[0, 1].data_ptr(), m=M))
    bgs = (L.SsBgStream * 1)(L.SsBgStream(slot=1, pool=cpools[("int16", "device")]._h.value,
                                          ids_dev=lay[1, 0].data_ptr(), offsets_dev=lay[1, 1].data_ptr(),
                                          heads_dev=lay[1, 2].data_ptr(), counts_dev=lay[1, 3].data_ptr(), m=M))
    nc = len(clips["int16"])
    sel = np.full(nc, 100, np.int32)
    neg = sel.copy()
    neg[3] = -1
    zero = np.zeros(nc, np.int32)

    def E(slot=0, r=None, total=48000, sr=RATE, s=None):
        return L.SsLayoutDraw(slot=slot, rng_dev=rng.data_ptr() if r is None else r, total=total, sample_rate=sr,
                              select_lengths=None if s is None else s.ctypes.data)

    def create(entries, count=None):
        arr = (L.SsLayoutDraw * len(entries))(*entries) if entries else None
        h = ctypes.c_void_p(12345)
        st = R.lib.ss_plan_create_layout(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0, strm, 1, bgs, 1,
                                         None, 0, arr, len(entries) if count is None else count, ctypes.byref(h))
        if st == L.SS_OK:
            R.lib.ss_plan_destroy(h)
            return st
        assert h.value == 12345                                    # *out untouched
        return st

    assert create([E(0), E(1, s=sel)]) == L.SS_OK
    assert create([]) == L.SS_OK                                   # ss_plan_create_lufs
    invalid = [[E(2)], [E(3)], [E(-1)], [E(0), E(0)], [E(r=0)], [E(r=rng.data_ptr() + 4)], [E(total=0)], [E(sr=0)],
               [E(sr=(1 << 31) // 10 + 1)], [E(0, s=sel)], [E(1, s=neg)],
               [E(r=lay[0, 0].data_ptr())],                       # rng over a layout the plan writes
               [E(r=o[0].data_ptr())]]                            # ... over an output
    for b in invalid:
        assert create(b) == L.SS_ERR_INVALID, b
    assert create([E()], count=-1) == L.SS_ERR_INVALID
    assert create([E(1, total=100000, s=zero)]) == L.SS_OK        # K = n: 9 clips
    many = R.dry_pool([np.ones(1, np.int16)] * 1100, dtype="int16")
    strm[0].pool = many._h.value
    assert create([E(0, total=1024)]) == L.SS_OK
    assert create([E(0, total=1025)]) == L.SS_ERR_UNSUPPORTED
    strm[0].pool = upools["device"]._h.value
    # a drawn layout meeting another range: the stream's offsets are the bed's ids
    strm[0].offsets_dev = lay[1, 0].data_ptr()
    assert create([E(0)]) == L.SS_ERR_INVALID
    assert create([E(1)]) == L.SS_ERR_INVALID
    strm[0].offsets_dev = lay[0, 1].data_ptr()
    h = ctypes.c_void_p()
    assert R.lib.ss_plan_create_layout(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0, strm, 1, bgs, 1,
                                       None, 0, None, 1, ctypes.byref(h)) == L.SS_ERR_INVALID and not h.value
    many.close()


# -------------------------------------------------------------------------------------------------------- scale
def test_hundreds_of_draws_over_thousands_of_utterances():
    from sonicsim_b200 import dry
    render, R = _R()
    rng = np.random.default_rng(12)
    utts = [np.clip(np.round(rng.standard_normal(int(k)) * 8000), -32768, 32767).astype(np.int16)
            for k in rng.integers(25, 65, 3000)]
    lengths = [u.size for u in utts]
    total = 30000
    K = dry.long_audio_max_selected(lengths, total)
    assert 800 <= K <= 1024
    cands = static_equal_n(1201, n=2, N=20000)
    pool = R.source_pool([c.src for c in cands])
    up = R.dry_pool(utts, dtype="int16")
    S, m, wl = 300, 128, 2000
    d = "cuda"
    picks = torch.from_numpy(rng.integers(0, 2, S).astype(np.int32)).to(d)
    lays = [torch.full((2, S, m), -1, dtype=torch.int32, device=d) for _ in range(2)]
    rng_t = torch.tensor([-77, 123456789], dtype=torch.int64, device=d)
    outs = [[torch.empty((2, wl), device=d) for _ in range(S)] for _ in range(2)]
    plans = []
    starts = rng.integers(0, 20000 - wl, S).tolist()
    try:
        for arm in range(2):
            srcs = [render.Pooled(pool, picks[j:j + 1], (starts[j], wl), 0,
                                  render.DryStream(up, lays[arm][0, j], lays[arm][1, j])) for j in range(S)]
            plans.append(R.plan_device(srcs, outs[arm], layouts=[render.LayoutDraw(j, rng_t, total, 1)
                                                                  for j in range(S)] if arm == 0 else None))
        for t in (0, 1):
            rng_t[1] += t
            plans[0].run()
            torch.cuda.synchronize()
            R.check_device_errors()
            got = lays[0].cpu().numpy()
            seed_t = rng_t.cpu().numpy()
            for j in range(0, S, 7):
                want = emu_rows(seed_t, j, lengths, total, m, 1, False)
                assert np.array_equal(got[0, j], want[0]) and np.array_equal(got[1, j], want[1]), (t, j)
            assert ((got[0] >= 0).sum(axis=1) == m).all()      # every row reaches the m = 128 cut
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
