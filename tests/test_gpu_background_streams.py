"""Background streams (render.BackgroundStream; ss_plan_create_bg) through the real kernels.  Every plan is run twice on
the same picks, starts, variates, SIRs and SNRs: once with bed slots, whose layouts (ids, offsets, heads, counts) change
at every run with no re-plan, and once with the same slots dry-picking, from a dry pool of the same dtype, the beds those
layouts lay out, assembled on the host to the slot pool's longest N (of the same residency; a float32 host pool where a
host source pool refuses a float32 device one).  Checked, bit for bit:
  1. stems and direct stems over float32 and 16-bit clip pools x device and host clip pools x device, host and tap-form
     host source pools, over several runs, one of them on a side stream behind queued work;
  2. training steps whose noise slot is a bed: a start draw whose readers include the bed slot, mixtures per channel
     with noise_delay and dereverberation targets and mono, speakers_out, rms_db, drawn starts and `used`;
  3. a bed laid out from the entries of the reference-order dry.create_background_audio equals a pick of its output;
  4. invalid layout entries are skipped, with bit 5 raising ValueError from check_device_errors;
  5. a clip pool closed under a live plan; dry.background_audio_layouts on CUDA tensors without a host synchronisation;
  6. refusals in Python and through the C ABI, with no plan created."""
import ctypes
import gc
import json
import random

import numpy as np
import pytest
import torch

from gpu_plumbing import _R
from pool_worlds import _host_pool, noises, speakers

pytestmark = pytest.mark.gpu

TAPS = 40
NAN = float("nan")
RATE = 16000
SLEEP = int(5e8)
M = 12


def clip_signals(seed, n, lo, hi):
    """n clips of lo..hi samples as int16 and as float32 values (the float32 ones not 16-bit representable)."""
    rng = np.random.default_rng(seed)
    i16, f32 = [], []
    for _ in range(n):
        k = int(rng.integers(lo, hi + 1))
        v = np.cumsum(rng.standard_normal(k)) * 0.02 + rng.standard_normal(k)
        v *= rng.uniform(0.05, 0.9) / max(1e-9, np.abs(v).max())
        i16.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
        f32.append((v + rng.standard_normal(k) * 1e-6).astype(np.float32))
    return {"int16": i16, "float32": f32}


def walk(ids, offs, heads, counts, lengths):
    kept, bad, end = [], False, 0
    for i, o, h, c in zip(ids, offs, heads, counts):
        if i < 0:
            continue
        if i >= len(lengths) or o < 0 or h < 0 or c < 1 or h + c > lengths[i] or o < end:
            bad = True
            continue
        kept.append((int(i), int(o), int(h), int(c)))
        end = o + c
    return kept, bad


def assemble(lay, clips, cut):
    """The bed of `cut` samples a layout (ids, offsets, heads, counts) lays out, in the clips' dtype."""
    k = np.zeros(cut, clips[0].dtype)
    for i, o, h, c in walk(*lay, [x.size for x in clips])[0]:
        if o < cut:
            n = min(c, cut - o)
            k[o:o + n] = clips[i][h:h + n]
    return k


def random_layouts(rng, k, lengths, cut, invalid=False):
    """k layouts of M entries: clip spans (whole, or cut at either end) behind gaps of 0..1 s from a random start, a few
    empty entries, the last reaching past cut; with `invalid`, some entries invalid."""
    lay = np.full((4, k, M), -1, np.int32)
    n = len(lengths)
    for j in range(k):
        pos, e = int(rng.integers(-RATE // 2, RATE // 2)), 0
        while e < M and pos < cut + RATE:
            if rng.random() < 0.1:
                e += 1
                continue
            i = int(rng.integers(0, n))
            L = lengths[i]
            h = int(rng.integers(0, L)) if rng.random() < 0.4 else 0
            c = int(rng.integers(1, L - h + 1)) if rng.random() < 0.4 else L - h
            o = max(0, pos)
            lay[:, j, e] = i, o, h, c
            if invalid and rng.random() < 0.2:
                q = int(rng.integers(0, 6))
                lay[:, j, e] = [(n, o, h, c), (i, -2, h, c), (i, o, -1, c), (i, o, h, 0), (i, o, h, L - h + 1),
                                (i, o - 1, h, c) if o > 0 else (i, -1, h, c)][q]
            pos = o + c + int(rng.integers(0, RATE))
            e += 1
    return lay


def twin_resident(clip_res, src_res, dtype):
    return "host" if src_res != "device" and dtype == "float32" else clip_res


def make_pool(R, clips, dtype, resident, levels=False):
    host = resident == "host"
    if dtype == "float32" and not host:
        clips = [torch.from_numpy(c).cuda() for c in clips]
    return R.dry_pool(clips, levels=levels, host=host, dtype=dtype)


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    spk = speakers(801, n=4, taps=TAPS)
    noi = noises(802, n=3)
    tap_banks = [R.rir_bank(c.h, False, TAPS, host=True, form="taps") for c in spk]
    pools = {"device": R.source_pool([c.src for c in spk]),
             "host": _host_pool(R, render, spk, TAPS),
             "taps": R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(spk, tap_banks)])}
    npools = {"device": R.source_pool([c.src for c in noi]), "host": _host_pool(R, render, noi)}
    clips = clip_signals(803, 7, 1, int(1.3 * RATE))
    for v in clips.values():
        v[2] = v[2][:1]                                            # a one-sample clip
    cpools = {(d, r): make_pool(R, clips[d], d, r) for d in clips for r in ("device", "host")}
    yield spk, noi, pools, npools, clips, cpools
    for p in list(pools.values()) + list(npools.values()) + list(cpools.values()):
        p.close()
    for b in tap_banks:
        b.close()


class Arms:
    """k pooled slots over one pool: bed slots (layout rows) and their twins dry-picking the assembled beds."""

    def __init__(self, R, render, pool, cpool, cands, wl, taps, k=4):
        self.k, self.wl, self.taps, self.cands = k, wl, taps, cands
        d = "cuda"
        self.picks = torch.zeros(k, dtype=torch.int32, device=d)
        self.starts = torch.zeros(k, dtype=torch.int32, device=d)
        self.lay = torch.full((4, k, M), -1, dtype=torch.int32, device=d)
        self.dpicks = torch.arange(k, dtype=torch.int32, device=d)
        C = cands[0].C
        self.outs = [torch.empty((C, wl), device=d) for _ in range(2 * k)]
        self.douts = [torch.empty((C, wl), device=d) for _ in range(2 * k)] if taps else None
        self.srcs = [render.Pooled(pool, self.picks[j], (self.starts[j], wl), taps,
                                   render.BackgroundStream(cpool, *[self.lay[q, j] for q in range(4)]))
                     for j in range(k)]
        self.plan = R.plan_device(self.srcs, self.outs[:k], direct_outs=self.douts[:k] if taps else None)
        self.pool, self.render, self.R = pool, render, R

    def oracle(self, beds, dtype, resident):
        apool = make_pool(self.R, beds, dtype, resident)
        srcs = [self.render.Pooled(self.pool, self.picks[j], (self.starts[j], self.wl), self.taps,
                                   self.render.DryPick(apool, self.dpicks[j])) for j in range(self.k)]
        plan = self.R.plan_device(srcs, self.outs[self.k:], direct_outs=self.douts[self.k:] if self.taps else None)
        return apool, plan

    def pairs(self):
        k = self.k
        return list(zip(self.outs[:k] + (self.douts or [])[:k], self.outs[k:] + (self.douts or [])[k:]))


# ------------------------------------------------------------------------------------------------ 1. stems
@pytest.mark.parametrize("src_resident", ["device", "host", "taps"])
@pytest.mark.parametrize("clip_resident", ["device", "host"])
@pytest.mark.parametrize("dtype", ["float32", "int16"])
def test_stems_equal_the_assembled_pick(world, dtype, clip_resident, src_resident):
    render, R = _R()
    spk, _, pools, _, clips, cpools = world
    cl = clips[dtype]
    lengths = [c.size for c in cl]
    cut, n_min = max(c.N for c in spk), min(c.N for c in spk)
    wl = 9000
    A = Arms(R, render, pools[src_resident], cpools[(dtype, clip_resident)], spk, wl, TAPS)
    rng = np.random.default_rng([len(dtype), len(clip_resident), len(src_resident)])
    side = torch.cuda.Stream()
    try:
        for run in range(3):
            lay = random_layouts(rng, A.k, lengths, cut)
            if run == 0:                                  # a bed wholly of gaps
                lay[:, 0] = -1
            A.lay.copy_(torch.from_numpy(lay))
            A.picks.copy_(torch.from_numpy(rng.integers(0, len(spk), A.k).astype(np.int32)))
            A.starts.copy_(torch.from_numpy(rng.integers(0, n_min - wl + 1, A.k).astype(np.int32)))
            if run == 0:
                A.picks.fill_(int(np.argmax([c.N for c in spk])))
                A.starts.copy_(torch.tensor([0, cut - wl, cut - wl, 0], dtype=torch.int32))
            beds = [assemble(lay[:, j], cl, cut) for j in range(A.k)]
            apool, oplan = A.oracle(beds, dtype, twin_resident(clip_resident, src_resident, dtype))
            for x, y in A.pairs():
                x.fill_(NAN)
                y.fill_(NAN)
            if run == 1:                                  # on a side stream behind queued work
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    torch.cuda._sleep(SLEEP)
                    A.plan.run(stream=side.cuda_stream)
                    oplan.run(stream=side.cuda_stream)
                    assert not side.query()
                torch.cuda.current_stream().wait_stream(side)
            else:
                A.plan.run()
                oplan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            for j, (x, y) in enumerate(A.pairs()):
                assert torch.isfinite(x).all() and torch.equal(x, y), (run, j)
            oplan.close()
            apool.close()
        assert A.plan.is_graph()
    finally:
        A.plan.close()


# ------------------------------------------------------------------------------------------- 2. draws and mixtures
LEN = RATE


class Step:
    """B examples: two speakers (plain pooled slots with direct targets), a noise slot that is a bed (or its twin's dry
    pick); one CropDraw over both speakers whose readers include the noise slot, one mixture per channel with
    noise_delay and dereverberation targets and one mono."""

    def __init__(self, R, render, sp, npool, B, noise_of, thr=-35.0, tries=37, delay=1234):
        d = "cuda"
        self.B = B
        self.picks = torch.zeros((B, 3), dtype=torch.int32, device=d)
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.u = torch.zeros((B, tries), dtype=torch.float64, device=d)
        self.used = torch.full((B,), -7, dtype=torch.int32, device=d)
        self.sirs = torch.zeros((B, 1), device=d)
        self.snr = torch.zeros(B, device=d)
        self.outs = [torch.empty((2, LEN), device=d) for _ in range(3 * B)]
        self.douts = [torch.empty((2, LEN), device=d) if j % 3 < 2 else None for j in range(3 * B)]
        self.mix = torch.empty((B, 2, LEN), device=d)
        self.spo = torch.empty((B, 2, 2, LEN), device=d)
        self.tgt = torch.empty((B, 2, 2, LEN), device=d)
        self.rms = torch.empty((B, 2), device=d)
        self.mmix = torch.empty((B, LEN), device=d)
        self.mspo = torch.empty((B, 2, LEN), device=d)
        self.mrms = torch.empty((B, 2), device=d)
        srcs, draws, mixes = [], [], []
        for b in range(B):
            w = (self.starts[b], LEN)
            srcs += [render.Pooled(sp, self.picks[b, 0], w, TAPS), render.Pooled(sp, self.picks[b, 1], w, TAPS),
                     render.Pooled(npool, self.picks[b, 2], w, 0, noise_of(b))]
            draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], self.u[b], self.used[b], thr))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mix[b],
                                        self.spo[b], self.rms[b], noise_delay=delay, direct_out=self.tgt[b]))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mmix[b],
                                        self.mspo[b], self.mrms[b], mono=True))
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts, mixtures=mixes, draws=draws)

    def tensors(self):
        return self.outs + [d for d in self.douts if d is not None] + [self.mix, self.spo, self.tgt, self.rms,
                                                                        self.mmix, self.mspo, self.mrms]

    def clear(self):
        for t in self.tensors():
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)


@pytest.mark.parametrize("src_resident", ["device", "host"])
@pytest.mark.parametrize("dtype", ["float32", "int16"])
def test_draws_and_mixtures_equal_the_assembled_pick(world, dtype, src_resident):
    render, R = _R()
    spk, noi, _, npools, clips, cpools = world
    cl = clips[dtype]
    lengths = [c.size for c in cl]
    sp = R.source_pool([c.src for c in spk], levels="mono")
    cut = max(c.N for c in noi)
    B = 6
    lay = torch.full((4, B, M), -1, dtype=torch.int32, device="cuda")
    S = Step(R, render, sp, npools[src_resident], B,
             lambda b: render.BackgroundStream(cpools[(dtype, "host")], *[lay[q, b] for q in range(4)]))
    rng = np.random.default_rng(91 + len(dtype) + len(src_resident))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    try:
        for run in range(3):
            h = random_layouts(rng, B, lengths, cut)
            lay.copy_(torch.from_numpy(h))
            apool = make_pool(R, [assemble(h[:, b], cl, cut) for b in range(B)], dtype, "host")
            dp = torch.arange(B, dtype=torch.int32, device="cuda")
            T = Step(R, render, sp, npools[src_resident], B, lambda b: render.DryPick(apool, dp[b]))
            S.picks[:, :2].copy_(torch.randint(0, len(spk), (B, 2), generator=gen, device="cuda", dtype=torch.int32))
            S.picks[:, 2].copy_(torch.randint(0, len(noi), (B,), generator=gen, device="cuda", dtype=torch.int32))
            S.u.uniform_(generator=gen)
            S.sirs.uniform_(-6, 6, generator=gen)
            S.snr.uniform_(5, 20, generator=gen)
            for a, b in ((T.picks, S.picks), (T.u, S.u), (T.sirs, S.sirs), (T.snr, S.snr)):
                a.copy_(b)
            S.clear()
            T.clear()
            S.plan.run()
            T.plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            for j, (x, y) in enumerate(zip(S.tensors() + [S.starts, S.used], T.tensors() + [T.starts, T.used])):
                assert torch.equal(x, y), (run, j)
            assert torch.isfinite(S.mix).all()
            T.plan.close()
            apool.close()
    finally:
        S.plan.close()
        sp.close()


# --------------------------------------------------------------------------- 3. against create_background_audio
def test_bed_equals_create_background_audio(world, tmp_path):
    """Seeded `random`: dry.create_background_audio (fake loader: 44.1 kHz stereo and 16 kHz mono clips) builds a bed;
    the same seed replayed through get_random_wav_path_from_json + _place_background_audio gives the entries, which a
    bed slot over a float32 pool of dry.background_clips renders bit for bit as a pick of the function's output."""
    from sonicsim_b200 import dry
    render, R = _R()
    spk, _, pools, _, _, _ = world
    rng = np.random.default_rng(17)
    raw = {}
    for j in range(6):
        if j % 2:
            raw["c%d.wav" % j] = (torch.from_numpy(rng.standard_normal((2, int(rng.integers(20000, 60000))))
                                                  .astype(np.float32) * 0.3), 44100)
        else:
            raw["c%d.wav" % j] = (torch.from_numpy(rng.standard_normal((1, int(rng.integers(8000, 20000))))
                                                  .astype(np.float32) * 0.3), RATE)
    js = tmp_path / "bg.json"
    js.write_text(json.dumps({p: int(w.shape[-1]) for p, (w, _) in raw.items()}))
    loader = lambda p: (raw[p][0].clone(), raw[p][1])        # noqa: E731
    paths = list(raw)
    clips = [c.numpy() for c in dry.background_clips(paths, RATE, loader)]
    cpool = R.dry_pool([torch.from_numpy(c).cuda() for c in clips])
    cut = max(c.N for c in spk)
    length = (cut - 100) / RATE
    total = int(length * RATE)                           # the bed's samples, padded with zeros to the slot pool's cut
    A = Arms(R, render, pools["device"], cpool, spk, 9000, TAPS, k=4)
    try:
        beds, lays = [], np.full((4, A.k, M), -1, np.int32)
        for j in range(A.k):
            random.seed(1000 + j)
            bed, _, _ = dry.create_background_audio(str(js), length, RATE, loader=loader)
            assert bed.shape == (1, total)
            beds.append(np.concatenate([bed[0].numpy(), np.zeros(cut - total, np.float32)]))
            random.seed(1000 + j)
            chosen = dry.get_random_wav_path_from_json(str(js), total, threshold=0.4)
            places, _, _ = dry._place_background_audio([clips[paths.index(p)].size for p in chosen], total, length,
                                                       RATE)
            assert places
            for e, (k, dst, src, count) in enumerate(places):
                lays[:, j, e] = paths.index(chosen[k]), dst, src, count
        A.lay.copy_(torch.from_numpy(lays))
        A.picks.copy_(torch.arange(A.k, dtype=torch.int32) % len(spk))
        A.starts.copy_(torch.tensor([0, 1000, cut - 9000, 5000], dtype=torch.int32).clamp(
            max=min(c.N for c in spk) - 9000))
        apool, oplan = A.oracle([b.astype(np.float32) for b in beds], "float32", "device")
        A.plan.run()
        oplan.run()
        torch.cuda.synchronize()
        R.check_device_errors()
        for j, (x, y) in enumerate(A.pairs()):
            assert torch.isfinite(x).all() and torch.equal(x, y), j
        oplan.close()
        apool.close()
    finally:
        A.plan.close()
        cpool.close()


# --------------------------------------------------------------------------------------------------- 4. bit 5
def test_invalid_entries_are_skipped_and_reported(world):
    render, R = _R()
    spk, _, pools, _, clips, cpools = world
    cl = clips["float32"]
    lengths = [c.size for c in cl]
    cut, n_min = max(c.N for c in spk), min(c.N for c in spk)
    A = Arms(R, render, pools["device"], cpools[("float32", "device")], spk, 8000, TAPS)
    rng = np.random.default_rng(57)
    try:
        lay = random_layouts(rng, A.k, lengths, cut, invalid=True)
        assert any(walk(*lay[:, j], lengths)[1] for j in range(A.k))
        A.lay.copy_(torch.from_numpy(lay))
        A.starts.copy_(torch.from_numpy(rng.integers(0, n_min - 8000 + 1, A.k).astype(np.int32)))
        kept = np.full_like(lay, -1)                     # the twin: the same layouts without the invalid entries
        for j in range(A.k):
            for e, v in enumerate(walk(*lay[:, j], lengths)[0]):
                kept[:, j, e] = v
        apool, oplan = A.oracle([assemble(kept[:, j], cl, cut) for j in range(A.k)], "float32", "device")
        A.plan.run()
        oplan.run()
        with pytest.raises(ValueError, match="BackgroundStream"):
            R.check_device_errors()
        for x, y in A.pairs():
            assert torch.equal(x, y)
        A.lay.copy_(torch.from_numpy(random_layouts(rng, A.k, lengths, cut)))
        A.plan.run()
        R.check_device_errors()
        oplan.close()
        apool.close()
    finally:
        A.plan.close()


# ------------------------------------------------------------------------------------------- 5. pool life, syncs
def test_clip_pool_closed_under_a_live_plan(world):
    render, R = _R()
    spk, _, pools, _, clips, _ = world
    cl = [np.tile(c, 1 + (40 * RATE) // c.size)[:40 * RATE] for c in clips["float32"][:5]] * 4
    cp = R.dry_pool(cl, host=True)
    A = Arms(R, render, pools["device"], cp, spk, 9000, TAPS)
    rng = np.random.default_rng(61)
    try:
        A.lay.copy_(torch.from_numpy(random_layouts(rng, A.k, [c.size for c in cl], max(c.N for c in spk))))
        A.plan.run()
        torch.cuda.synchronize()
        before = [x.clone() for x, _ in A.pairs()]
        cp.close()
        assert cp.closed and cp._h.value and cp._plans == 1
        with pytest.raises(ValueError, match="is closed"):
            R.plan_device([render.Pooled(pools["device"], A.picks[0], (A.starts[0], 9000), TAPS,
                                         render.BackgroundStream(cp, *[A.lay[q, 0] for q in range(4)]))],
                          [torch.empty((2, 9000), device="cuda")])
        for x, _ in A.pairs():
            x.fill_(NAN)
        A.plan.run()
        torch.cuda.synchronize()
        for b, (x, _) in zip(before, A.pairs()):
            assert torch.equal(b, x)
        R.check_device_errors()
        A.plan.close()
        gc.collect()
        assert not cp._h.value and cp._plans == 0
    finally:
        A.plan.close()
        cp.close()


def test_layouts_without_host_synchronisation():
    from sonicsim_b200 import dry
    lengths = torch.randint(RATE, 60 * RATE, (1000,), device="cuda", dtype=torch.int32)
    sel = (lengths.long() * 441) // 160
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    dry.background_audio_layouts(lengths, 10 * RATE, 8, 4, generator=gen)     # warm-up
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = dry.background_audio_layouts(lengths, 10 * RATE, 8, 128, generator=gen, select_lengths=sel)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert all(t.shape == (128, 8) and t.dtype == torch.int32 and t.is_cuda for t in out)
    assert bool((out[0][:, 0] >= 0).all())


# ------------------------------------------------------------------------------------------------- 6. refusals
def test_python_refusals(world):
    render, R = _R()
    spk, _, pools, _, clips, cpools = world
    pool, cp = pools["device"], cpools[("float32", "device")]
    lay = [torch.full((M,), -1, dtype=torch.int32, device="cuda") for _ in range(4)]
    pick, start = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    o = [torch.empty((2, 4000), device="cuda")]

    def bg(*a, p=cp):
        v = list(lay)
        for q, t in a:
            v[q] = t
        return render.BackgroundStream(p, *v)

    gp = R.source_pool([c.src for c in spk], lufs_targets=[-20.0] * len(spk))
    lp = R.source_pool([c.src for c in spk], levels="mono")
    closed = make_pool(R, clips["float32"], "float32", "device")
    closed.close()
    try:
        for d, p, match in [
            (bg(), gp, "loudness gains"),
            (bg((0, lay[0].long())), pool, "int32"),
            (bg((2, lay[2].long())), pool, "int32"),
            (bg((1, lay[1][:5])), pool, "shape"),
            (bg((3, lay[3][:5])), pool, "shape"),
            (bg((3, lay[3].cpu())), pool, "CUDA"),
            (bg((0, torch.full((129,), -1, dtype=torch.int32, device="cuda"))), pool, "1 to 128"),
            (bg((0, lay[0][:0])), pool, "1 to 128"),
            (bg((0, lay[0].reshape(3, 4))), pool, "shape"),
            (bg((2, torch.full((2 * M,), -1, dtype=torch.int32, device="cuda")[::2])), pool, "contiguous"),
            (bg(p="pool"), pool, "DryPool"),
            (bg(p=closed), pool, "is closed"),
        ]:
            with pytest.raises(ValueError, match=match):
                R.plan_device([render.Pooled(p, pick, (start, 4000), 0, d)], o)
        u = torch.rand(5, dtype=torch.float64, device="cuda")
        with pytest.raises(ValueError, match="bed slot"):
            R.plan_device([render.Pooled(lp, pick, (start, 4000), 0, bg())], o, draws=[render.CropDraw(start, [0], u)])
        with pytest.raises(ValueError, match="not a pooled slot"):
            R.plan_device([spk[0].src._replace(window=(0, 4000), dry=bg())], o)
        # DryStream keeps refusing float32 pools
        with pytest.raises(ValueError, match="16-bit"):
            R.plan_device([render.Pooled(pool, pick, (start, 4000), 0, render.DryStream(cp, lay[0], lay[1]))], o)
        # accepted: a bed slot that reads a draw's start beside a speaker
        R.plan_device([render.Pooled(lp, pick, (start, 4000), 0), render.Pooled(lp, pick, (start, 4000), 0, bg())],
                      o + [torch.empty((2, 4000), device="cuda")], draws=[render.CropDraw(start, [0], u)]).close()
    finally:
        gp.close()
        lp.close()


def test_c_abi_refusals(world):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    spk, _, pools, _, clips, cpools = world
    pool, cp = pools["device"], cpools[("int16", "device")]
    lay = torch.full((4, M + 1), -1, dtype=torch.int32, device="cuda")
    pick = torch.zeros(2, dtype=torch.int32, device="cuda")
    o = [torch.empty((2, 4000), device="cuda") for _ in range(2)]
    items, n, keep = R._device_items([render.Pooled(pool, pick[j:j + 1], (0, 4000), 0) for j in range(2)], o)
    ptr = [lay[q].data_ptr() for q in range(4)]
    try:
        def create(bgs, picks=None, streams=None, mixes=None, draws=None, items_=None, n_bgs=None):
            arr = (L.SsBgStream * len(bgs))(*bgs) if bgs else None
            pk = (L.SsDryPick * len(picks))(*picks) if picks else None
            sa = (L.SsDryStream * len(streams))(*streams) if streams else None
            h = ctypes.c_void_p(0x5A5A)
            its, ni = items_ if items_ is not None else (items, n)
            st = R.lib.ss_plan_create_bg(R.ctx, its, ni, mixes, len(mixes) if mixes else 0, draws,
                                         len(draws) if draws else 0, pk, None, len(picks) if picks else 0, None, 0,
                                         sa, len(streams) if streams else 0, arr,
                                         len(bgs) if n_bgs is None else n_bgs, ctypes.byref(h))
            if st == L.SS_OK:
                R.lib.ss_plan_destroy(h)
            else:
                assert h.value == 0x5A5A                  # a refused call leaves *out untouched
            return st

        def G(slot=0, pool_h=None, a=None, m=M):
            a = list(ptr) if a is None else a
            return L.SsBgStream(slot=slot, pool=pool_h if pool_h is not None else cp._h.value, ids_dev=a[0],
                                offsets_dev=a[1], heads_dev=a[2], counts_dev=a[3], m=m)

        def P(q, v):
            a = list(ptr)
            a[q] = v
            return a

        assert create([G()]) == L.SS_OK
        assert create([G(pool_h=cpools[("float32", "host")]._h.value)]) == L.SS_OK
        assert create([]) == L.SS_OK                      # no beds: ss_plan_create_stream
        bad = [[G(slot=2)], [G(slot=-1)], [G(), G()], [G(m=0)], [G(m=129)], [G(pool_h=0)]]
        bad += [[G(a=P(q, 0))] for q in range(4)] + [[G(a=P(q, ptr[q] + 2))] for q in range(4)]
        for b in bad:
            assert create(b) == L.SS_ERR_INVALID, b
        assert create([G()], n_bgs=-1) == L.SS_ERR_INVALID
        assert create([], n_bgs=1) == L.SS_ERR_INVALID    # NULL bgs with n_bgs > 0
        apool = R.dry_pool([torch.zeros(max(c.N for c in spk), device="cuda")])
        up = cpools[("int16", "device")]
        try:
            assert create([G()], picks=[L.SsDryPick(slot=0, pool=apool._h.value, pick_dev=pick.data_ptr())]) == \
                L.SS_ERR_INVALID
            assert create([G()], streams=[L.SsDryStream(slot=0, pool=up._h.value, ids_dev=ptr[0], offsets_dev=ptr[1],
                                                        m=M)]) == L.SS_ERR_INVALID
        finally:
            apool.close()
        # a mixture writing over any of the four arrays
        for q in range(4):
            snr = torch.zeros(1, device="cuda")
            mx = (L.SsPlanMix * 1)()
            mx[0].speakers[0], mx[0].noises[0], mx[0].S, mx[0].M = 1, 0, 1, 1
            mx[0].snr, mx[0].mix = snr.data_ptr(), ptr[q]
            assert create([G()], mixes=mx) == L.SS_ERR_INVALID, q
        # a dry pool of another context
        ctx2 = ctypes.c_void_p()
        L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
        R2 = render.Renderer(R.device)
        R2.ctx = ctx2
        foreign = R2.dry_pool(clips["int16"], dtype="int16")
        try:
            assert create([G(pool_h=foreign._h.value)]) == L.SS_ERR_INVALID
        finally:
            foreign.close()
            R2.lib.ss_destroy(ctx2)
        # a slot that is not pooled, and a slot of a pool with loudness gains
        gp = R.source_pool([c.src for c in spk], lufs_targets=[-20.0] * len(spk))
        try:
            items2, n2, keep2 = R._device_items([spk[0].src._replace(window=(0, 4000)),
                                                 render.Pooled(gp, pick[1:2], (0, 4000), 0)], o)
            assert create([G(slot=0)], items_=(items2, n2)) == L.SS_ERR_INVALID
            assert create([G(slot=1)], items_=(items2, n2)) == L.SS_ERR_INVALID
        finally:
            gp.close()
        # a draw speaker is refused; a draw reader is accepted
        lp = R.source_pool([c.src for c in spk], levels="mono")
        start = torch.zeros(1, dtype=torch.int32, device="cuda")
        u = torch.rand(5, dtype=torch.float64, device="cuda")
        try:
            items3, n3, keep3 = R._device_items([render.Pooled(lp, pick[j:j + 1], (start, 4000), 0) for j in range(2)],
                                                o)
            dr = (L.SsPlanDraw * 1)()
            dr[0].start, dr[0].u, dr[0].S, dr[0].tries, dr[0].threshold_db = start.data_ptr(), u.data_ptr(), 1, 5, -40.0
            dr[0].speakers[0] = 0
            assert create([G(slot=0)], draws=dr, items_=(items3, n3)) == L.SS_ERR_INVALID
            assert create([G(slot=1)], draws=dr, items_=(items3, n3)) == L.SS_OK
        finally:
            lp.close()
    finally:
        pass
