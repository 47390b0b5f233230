"""Loudness slots (render.StemLoudness; ss_plan_create_lufs) through the real kernels.  A stream or bed slot with a
loudness target renders its whole stem at every run, measures it and stores its crop at the run's gain.  Every run
draws new layouts, picks, starts and targets into NaN-filled outputs, and each crop, direct crop and (LUFS, gain) is
compared, bit for bit, with the slice at the run's start of render_host(..., lufs_targets=[target]) of the picked
candidate with the stream or bed that run lays out; the LUFS also with the float64 BS.1770 oracle.  Checked:
  1. stream slots over 16-bit utterance pools and bed slots over float32 and 16-bit clip pools, device and host
     resident, over aligned speakers with direct stems, grid-blocked long RIRs and static noise; one run on a side stream;
  2. a training plan (draws, mixtures with noise_delay and dereverberation targets) keeps the starts and `used` of the
     same plan without targets, and its mixtures are the mixture kernels' on the normalised crops;
  3. a layout that reproduces a dry pool signal gets that pair's PairGains loudness and gain, bit for bit;
  4. a silent layout is measured -inf and gained as -40 LUFS; a non-finite target leaves the slot unscaled and raises
     ValueError from check_device_errors;
  5. launch counts: 7 more per run with targets, none without;
  6. refusals in Python and through the C ABI, with no plan created."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from gpu_plumbing import _R
from mix_reference import _rms_db, compose_mix, mix_gains_f64
from pool_worlds import Cand, _host_pool, speakers

pytestmark = pytest.mark.gpu

RATE = 16000
N = 48000                    # every candidate of a loudness slot's pool has one N
WL = 16000
TAPS = 40
M = 12
NAN = float("nan")
SLEEP = int(5e8)
DELAY = 1234


def equal_n_cands(seed, kind):
    """Candidates of one N: aligned speakers (direct stems), grid-blocked long RIRs, static noise."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(3):
        if kind == "static":
            out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 4096)[0], None))
            continue
        P = 3 + j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        if kind == "aligned":
            out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b, TAPS))
        else:
            out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 1, 9000), b))
    return out


def signals(seed, n, lo, hi):
    """n clips of lo..hi samples as int16 and as float32 values."""
    rng = np.random.default_rng(seed)
    i16, f32 = [], []
    for _ in range(n):
        k = int(rng.integers(lo, hi + 1))
        v = np.cumsum(rng.standard_normal(k)) * 0.02 + rng.standard_normal(k)
        v *= rng.uniform(0.05, 0.9) / max(1e-9, np.abs(v).max())
        i16.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
        f32.append((v + rng.standard_normal(k) * 1e-6).astype(np.float32))
    return {"int16": i16, "float32": f32}


def as_float(x):
    return x.astype(np.float32) * np.float32(1 / 32768) if x.dtype == np.int16 else x


def layout_stream(rng, lengths):
    """(ids, offsets) of M entries: utterances behind gaps of 0..1 s, a few empty entries, reaching past N."""
    ids, offs = np.full(M, -1, np.int32), np.full(M, -1, np.int32)
    pos, e = int(rng.integers(0, RATE)), 0
    while e < M and pos < N + RATE:
        if rng.random() < 0.1:
            e += 1
            continue
        i = int(rng.integers(0, len(lengths)))
        ids[e], offs[e] = i, pos
        pos += lengths[i] + int(rng.integers(0, RATE))
        e += 1
    return np.stack([ids, offs])


def layout_bed(rng, lengths):
    """(ids, offsets, heads, counts) of M entries: clip spans, whole or trimmed, behind gaps of 0..0.5 s."""
    lay = np.full((4, M), -1, np.int32)
    pos, e = int(rng.integers(0, RATE // 2)), 0
    while e < M and pos < N + RATE:
        i = int(rng.integers(0, len(lengths)))
        L = lengths[i]
        h = int(rng.integers(0, L)) if rng.random() < 0.4 else 0
        c = int(rng.integers(1, L - h + 1)) if rng.random() < 0.4 else L - h
        lay[:, e] = i, pos, h, c
        pos += c + int(rng.integers(0, RATE // 2))
        e += 1
    return lay


def assemble(lay, clips):
    """The first N samples of the stream a layout lays out, as float32 (float32 or int16 clips)."""
    out = np.zeros(N, np.float32)
    if lay.shape[0] == 2:
        lay = np.stack([lay[0], lay[1], np.zeros(M, np.int32), np.array([clips[i].size if i >= 0 else 0
                                                                          for i in lay[0]], np.int32)])
    end = 0
    for i, o, h, c in lay.T:
        if i < 0:
            continue
        assert o >= end and h + c <= clips[i].size         # (the layouts here are valid)
        end = o + c
        if o < N:
            n = min(c, N - o)
            out[o:o + n] = as_float(clips[i][h:h + n])
    return out


def reference(R, render, c, x, t, taps):
    """render_host of candidate c with dry x and target t: (whole stem, whole direct stem or None, (LUFS, gain), raw
    stem without a target)."""
    src = (render.MovingSource(x, c.bank, c.b, direct_taps=taps) if c.b is not None
           else render.StaticSource(x, c.bank))
    dout = [np.empty((c.C, N), np.float32)] if taps else None
    lo = []
    y = R.render_host([src], lufs_targets=[t], loudness_out=lo, sr=RATE, direct_outs=dout)[0]
    raw = R.render_host([src], direct_outs=[np.empty((c.C, N), np.float32)] if taps else None)[0]
    return y, (dout[0] if taps else None), tuple(lo[0]), raw


def oracle_lufs(raw):
    return so.bs1770_integrated_loudness(raw.T.astype(np.float64), RATE, 0.4, up_to_8_channels=True)


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    cands = {k: equal_n_cands(900 + j, k) for j, k in enumerate(("aligned", "grid", "static"))}
    pools = {k: R.source_pool([c.src for c in v]) for k, v in cands.items()}
    clips = signals(910, 7, 1, int(1.3 * RATE))
    clips["int16"][2] = clips["int16"][2][:1]
    utts = clips["int16"]
    upools = {r: R.dry_pool(utts, levels=True, host=r == "host", dtype="int16") for r in ("device", "host")}
    cpools = {(d, r): R.dry_pool(clips[d] if r == "host" or d == "int16" else [torch.from_numpy(v).cuda()
                                                                               for v in clips[d]],
                                 host=r == "host", dtype=d)
              for d in ("float32", "int16") for r in ("device", "host")}
    yield cands, pools, clips, upools, cpools
    for p in list(pools.values()) + list(upools.values()) + list(cpools.values()):
        p.close()


class Slots:
    """k stream or bed slots of one pool with loudness targets, device picks and starts, NaN-filled outputs."""

    def __init__(self, R, render, pool, cands, dpool, bed, taps, k=3, result=True):
        d = "cuda"
        self.k, self.taps, self.bed, self.cands = k, taps, bed, cands
        self.picks = torch.zeros(k, dtype=torch.int32, device=d)
        self.starts = torch.zeros(k, dtype=torch.int32, device=d)
        self.lay = torch.full((k, 4 if bed else 2, M), -1, dtype=torch.int32, device=d)
        self.lufs = torch.zeros((k, 1), dtype=torch.float64, device=d)
        self.res = torch.full((k, 2), NAN, dtype=torch.float64, device=d)
        C = cands[0].C
        self.outs = [torch.empty((C, WL), device=d) for _ in range(k)]
        self.douts = [torch.empty((C, WL), device=d) for _ in range(k)] if taps else None
        srcs = []
        for j in range(k):
            q = render.StemLoudness(self.lufs[j], self.res[j] if result else None, RATE)
            dry = (render.BackgroundStream(dpool, *[self.lay[j, r] for r in range(4)], lufs=q) if bed
                   else render.DryStream(dpool, self.lay[j, 0], self.lay[j, 1], lufs=q))
            srcs.append(render.Pooled(pool, self.picks[j], (self.starts[j], WL), taps, dry))
        self.srcs = srcs
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts)

    def draw(self, rng, clips):
        lays = np.stack([(layout_bed if self.bed else layout_stream)(rng, [c.size for c in clips])
                         for _ in range(self.k)])
        self.lay.copy_(torch.from_numpy(lays))
        self.picks.copy_(torch.from_numpy(rng.integers(0, len(self.cands), self.k).astype(np.int32)))
        s = rng.integers(0, N - WL + 1, self.k).astype(np.int32)
        s[0] = N - WL
        self.starts.copy_(torch.from_numpy(s))
        self.lufs.copy_(torch.from_numpy(rng.uniform(-31.0, -15.0, (self.k, 1))))
        for t in self.outs + (self.douts or []):
            t.fill_(NAN)
        self.res.fill_(NAN)
        return lays

    def check(self, R, render, lays, clips, oracle=True):
        picks, starts = self.picks.tolist(), self.starts.tolist()
        lufs, res = self.lufs.cpu().numpy()[:, 0], self.res.cpu().numpy()
        for j in range(self.k):
            c = self.cands[picks[j]]
            x = assemble(lays[j], clips)
            y, yd, lo, raw = reference(R, render, c, x, float(lufs[j]), self.taps)
            s = starts[j]
            assert torch.equal(self.outs[j].cpu(), torch.from_numpy(y[:, s:s + WL])), j
            if self.taps:
                assert torch.equal(self.douts[j].cpu(), torch.from_numpy(yd[:, s:s + WL])), j
            assert tuple(res[j]) == lo, (j, res[j], lo)
            if oracle and np.isfinite(lo[0]):
                assert abs(res[j, 0] - oracle_lufs(raw)) < 1e-6


# ------------------------------------------------------------------------------------------------ 1. stems
@pytest.mark.parametrize("u_resident", ["device", "host"])
@pytest.mark.parametrize("kind", ["aligned", "grid", "static"])
def test_stream_slots_equal_render_host_with_the_target(world, kind, u_resident):
    render, R = _R()
    cands, pools, clips, upools, _ = world
    taps = TAPS if kind == "aligned" else 0
    A = Slots(R, render, pools[kind], cands[kind], upools[u_resident], False, taps)
    rng = np.random.default_rng([len(kind), len(u_resident)])
    side = torch.cuda.Stream()
    try:
        for run in range(3):
            lays = A.draw(rng, clips["int16"])
            if run == 1:                                  # on a side stream behind queued work
                side.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(side):
                    torch.cuda._sleep(SLEEP)
                    A.plan.run(stream=side.cuda_stream)
                    assert not side.query()
                torch.cuda.current_stream().wait_stream(side)
            else:
                A.plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            A.check(R, render, lays, clips["int16"])
        assert A.plan.is_graph()
    finally:
        A.plan.close()


@pytest.mark.parametrize("c_resident", ["device", "host"])
@pytest.mark.parametrize("dtype", ["float32", "int16"])
def test_bed_slots_equal_render_host_with_the_target(world, dtype, c_resident):
    render, R = _R()
    cands, pools, clips, _, cpools = world
    rng = np.random.default_rng([len(dtype), len(c_resident)])
    for kind in ("static", "aligned"):
        taps = TAPS if kind == "aligned" else 0
        A = Slots(R, render, pools[kind], cands[kind], cpools[(dtype, c_resident)], True, taps,
                  result=kind == "static")
        try:
            for run in range(2):
                lays = A.draw(rng, clips[dtype])
                A.plan.run()
                torch.cuda.synchronize()
                R.check_device_errors()
                if kind == "static":
                    A.check(R, render, lays, clips[dtype])
                else:                                     # without a result tensor: the crops still carry the gain
                    A.res.fill_(NAN)
                    picks, starts, lufs = A.picks.tolist(), A.starts.tolist(), A.lufs.cpu().numpy()[:, 0]
                    for j in range(A.k):
                        y, yd, _, _ = reference(R, render, A.cands[picks[j]], assemble(lays[j], clips[dtype]),
                                                float(lufs[j]), taps)
                        s = starts[j]
                        assert torch.equal(A.outs[j].cpu(), torch.from_numpy(y[:, s:s + WL]))
                        assert torch.equal(A.douts[j].cpu(), torch.from_numpy(yd[:, s:s + WL]))
        finally:
            A.plan.close()


# ------------------------------------------------------------------------------------------ 2. training plans
class Step:
    """B examples: two stream speakers (aligned, direct stems) and a bed noise slot (static), one CropDraw over the
    speakers that the bed also reads, one mixture with noise_delay and dereverberation targets; `lufs` gives every slot
    a StemLoudness."""

    def __init__(self, R, render, world, B, lufs):
        cands, pools, clips, upools, cpools = world
        d = "cuda"
        self.B = B
        self.picks = torch.zeros((B, 3), dtype=torch.int32, device=d)
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.u = torch.zeros((B, 37), dtype=torch.float64, device=d)
        self.used = torch.zeros(B, dtype=torch.int32, device=d)
        self.lay = torch.full((B, 3, 4, M), -1, dtype=torch.int32, device=d)
        self.sirs = torch.zeros((B, 1), device=d)
        self.snr = torch.zeros(B, device=d)
        self.lufs = torch.zeros((B, 3), dtype=torch.float64, device=d)
        self.outs = [torch.empty((2, WL), device=d) for _ in range(3 * B)]
        self.douts = [torch.empty((2, WL), device=d) if j % 3 < 2 else None for j in range(3 * B)]
        self.mix = torch.empty((B, 2, WL), device=d)
        self.spo = torch.empty((B, 2, 2, WL), device=d)
        self.tgt = torch.empty((B, 2, 2, WL), device=d)
        self.rms = torch.empty((B, 2), device=d)
        srcs, draws, mixes = [], [], []
        for b in range(B):
            w = (self.starts[b], WL)
            q = [render.StemLoudness(self.lufs[b, k:k + 1]) if lufs else None for k in range(3)]
            for k in range(2):
                srcs.append(render.Pooled(pools["aligned"], self.picks[b, k], w, TAPS,
                                          render.DryStream(upools["device"], self.lay[b, k, 0], self.lay[b, k, 1],
                                                           lufs=q[k])))
            srcs.append(render.Pooled(pools["static"], self.picks[b, 2], w, 0,
                                      render.BackgroundStream(cpools[("float32", "device")],
                                                              *[self.lay[b, 2, r] for r in range(4)], lufs=q[2])))
            draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], self.u[b], self.used[b], -35.0))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mix[b],
                                        self.spo[b], self.rms[b], noise_delay=DELAY, direct_out=self.tgt[b]))
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts, mixtures=mixes, draws=draws)

    def fill(self, other):
        for a in ("picks", "u", "lay", "sirs", "snr", "lufs"):
            getattr(self, a).copy_(getattr(other, a))
        for t in self.outs + [x for x in self.douts if x is not None] + [self.mix, self.spo, self.tgt, self.rms]:
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)


def test_training_plan_keeps_starts_and_mixes_the_normalised_crops(world):
    render, R = _R()
    cands, pools, clips, upools, cpools = world
    B = 3
    A, Z = Step(R, render, world, B, True), Step(R, render, world, B, False)
    rng = np.random.default_rng(77)
    try:
        for run in range(2):
            lay = np.full((B, 3, 4, M), -1, np.int32)
            for b in range(B):
                for k in range(2):
                    lay[b, k, :2] = layout_stream(rng, [c.size for c in clips["int16"]])
                lay[b, 2] = layout_bed(rng, [c.size for c in clips["float32"]])
            A.lay.copy_(torch.from_numpy(lay))
            A.picks.copy_(torch.from_numpy(rng.integers(0, 3, (B, 3)).astype(np.int32)))
            A.u.uniform_()
            A.sirs.uniform_(-6, 6)
            A.snr.uniform_(10, 20)
            A.lufs.copy_(torch.from_numpy(np.stack([rng.uniform(-19, -15, B), rng.uniform(-19, -15, B),
                                                    rng.uniform(-26, -22, B)], 1)))
            Z.fill(A)
            A.fill(Z)
            A.plan.run()
            Z.plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            assert torch.equal(A.starts, Z.starts) and torch.equal(A.used, Z.used)
            starts, picks, lufs = A.starts.tolist(), A.picks.tolist(), A.lufs.cpu().numpy()
            for b in range(B):
                s = starts[b]
                for k in range(3):                         # the crops: render_host with the target
                    taps = TAPS if k < 2 else 0
                    c = cands["aligned" if k < 2 else "static"][picks[b][k]]
                    src = clips["int16"] if k < 2 else clips["float32"]
                    y, yd, _, _ = reference(R, render, c, assemble(lay[b, k] if k == 2 else lay[b, k, :2], src),
                                            float(lufs[b, k]), taps)
                    assert torch.equal(A.outs[3 * b + k].cpu(), torch.from_numpy(y[:, s:s + WL])), (run, b, k)
                    if taps:
                        assert torch.equal(A.douts[3 * b + k].cpu(), torch.from_numpy(yd[:, s:s + WL]))
                # the mixture on the normalised crops (per channel: the stems as they are): the mix reference's gains
                # and composition, speaker 0 and its target unscaled
                spk = np.stack([A.outs[3 * b + k].cpu().numpy().reshape(-1) for k in range(2)])
                noi = A.outs[3 * b + 2].cpu().numpy().reshape(1, -1)
                dirs = np.stack([A.douts[3 * b + k].cpu().numpy().reshape(-1) for k in range(2)])
                g, gn = mix_gains_f64(spk, noi, A.sirs[b].cpu().numpy(), float(A.snr[b]), DELAY)
                mix_ref, spo_ref = compose_mix(spk, noi, g.astype(np.float32), np.float32(gn), DELAY)
                mix, spo = A.mix[b].cpu().numpy().reshape(-1), A.spo[b].cpu().numpy().reshape(2, -1)
                tgt, rms = A.tgt[b].cpu().numpy().reshape(2, -1), A.rms[b].cpu().numpy()
                assert np.max(np.abs(mix - mix_ref)) <= 1e-5 * np.max(np.abs(mix_ref)), (run, b)
                assert np.array_equal(spo[0], spk[0]) and np.array_equal(tgt[0], dirs[0])
                assert np.max(np.abs(spo[1] - spo_ref[1])) <= 1e-6 * np.max(np.abs(spo_ref[1]))
                assert np.max(np.abs(tgt[1] - dirs[1] * np.float32(g[1]))) <= 1e-6 * np.max(np.abs(dirs[1] * g[1]))
                for k in range(2):
                    assert abs(rms[k] - _rms_db(spk[k])) < 1e-4
    finally:
        A.plan.close()
        Z.plan.close()


# ------------------------------------------------------------------------------------- 3. pair-gain cross-check
def test_a_layout_of_one_whole_signal_gets_its_pair_gain(world):
    render, R = _R()
    cands, pools, clips, upools, cpools = world
    rng = np.random.default_rng(5)
    sig = [np.clip(np.round(rng.standard_normal(N + 100 * j) * 3000), -32768, 32767).astype(np.int16)
           for j in range(2)]
    dp = R.dry_pool(sig, dtype="int16")
    t = rng.uniform(-19, -15, (2, 3))
    pg = R.pair_gains(pools["aligned"], dp, t, sr=RATE)
    A = Slots(R, render, pools["aligned"], cands["aligned"], dp, False, TAPS, k=2)
    try:
        for d in range(2):
            for i in range(3):
                lay = np.full((2, 2, M), -1, np.int32)
                lay[:, 0, 0], lay[:, 1, 0] = d, 0                 # signal d whole at offset 0
                A.lay.copy_(torch.from_numpy(lay))
                A.picks.fill_(i)
                A.starts.fill_(0)
                A.lufs.fill_(float(t[d, i]))
                A.plan.run()
                torch.cuda.synchronize()
                res = A.res.cpu().numpy()
                for j in range(2):
                    assert tuple(res[j]) == tuple(pg.loudness[d, i]), (d, i, res[j], pg.loudness[d, i])
    finally:
        A.plan.close()
        pg.close()
        dp.close()


# --------------------------------------------------------------------------------------- 4. silent and invalid
def test_silent_layout_and_non_finite_targets(world):
    render, R = _R()
    cands, pools, clips, upools, _ = world
    A = Slots(R, render, pools["aligned"], cands["aligned"], upools["device"], False, TAPS, k=3)
    rng = np.random.default_rng(9)
    try:
        lays = A.draw(rng, clips["int16"])
        lays[0][:] = -1                                            # no utterance at all
        A.lay[0].fill_(-1)
        A.lufs[0] = -24.0
        A.plan.run()
        torch.cuda.synchronize()
        R.check_device_errors()
        res = A.res.cpu().numpy()
        assert np.isneginf(res[0, 0]) and res[0, 1] == 10.0 ** ((-24.0 + 40.0) / 20.0)
        assert not A.outs[0].any()
        A.check(R, render, lays, clips["int16"])
        for bad in (NAN, math.inf, -math.inf):
            lays = A.draw(rng, clips["int16"])
            A.lufs[1] = bad
            A.plan.run()
            torch.cuda.synchronize()
            with pytest.raises(ValueError, match="not finite"):
                R.check_device_errors()
            R.check_device_errors()                                # (the bits were cleared)
            res = A.res.cpu().numpy()
            c = A.cands[A.picks[1].item()]
            _, _, lo, raw = reference(R, render, c, assemble(lays[1], clips["int16"]), -20.0, TAPS)
            s = A.starts[1].item()
            assert res[1, 0] == lo[0] and math.isnan(res[1, 1])
            assert torch.equal(A.outs[1].cpu(), torch.from_numpy(raw[:, s:s + WL]))       # unscaled
            for j in (0, 2):
                y, yd, lo, _ = reference(R, render, A.cands[A.picks[j].item()], assemble(lays[j], clips["int16"]),
                                         A.lufs[j].item(), TAPS)
                s = A.starts[j].item()
                assert torch.equal(A.outs[j].cpu(), torch.from_numpy(y[:, s:s + WL])) and tuple(res[j]) == lo
    finally:
        A.plan.close()


# --------------------------------------------------------------------------------------------- 5. launch counts
def test_launch_counts(world):
    render, R = _R()
    cands, pools, clips, upools, cpools = world

    def per_run(srcs, outs):
        plan = R.plan_device(srcs, outs)
        try:
            plan.run()
            torch.cuda.synchronize()
            before = R.launch_count()
            plan.run()
            plan.run()
            torch.cuda.synchronize()
            return (R.launch_count() - before) // 2
        finally:
            plan.close()

    ids = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    lay = torch.full((4, M), -1, dtype=torch.int32, device="cuda")
    pick = torch.zeros(1, dtype=torch.int32, device="cuda")
    t = torch.full((2,), -20.0, dtype=torch.float64, device="cuda")
    outs = [torch.empty((2, WL), device="cuda") for _ in range(2)]

    def srcs(with_lufs):
        q = [render.StemLoudness(t[k:k + 1]) if with_lufs else None for k in range(2)]
        return [render.Pooled(pools["aligned"], pick, (0, WL), 0, render.DryStream(upools["device"], ids, ids, q[0])),
                render.Pooled(pools["static"], pick, (100, WL), 0,
                              render.BackgroundStream(cpools[("int16", "host")], *lay, lufs=q[1]))]
    without, with_ = per_run(srcs(False), outs), per_run(srcs(True), outs)
    assert with_ == without + 7, (without, with_)
    one = per_run(srcs(True)[:1], outs[:1])
    assert one == per_run(srcs(False)[:1], outs[:1]) + 7


# -------------------------------------------------------------------------------------------------- 6. refusals
def test_python_refusals(world):
    render, R = _R()
    cands, pools, clips, upools, cpools = world
    up = upools["device"]
    ids = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    pick = torch.zeros(1, dtype=torch.int32, device="cuda")
    t = torch.full((4,), -20.0, dtype=torch.float64, device="cuda")
    res = torch.zeros(8, dtype=torch.float64, device="cuda")
    out = [torch.empty((2, WL), device="cuda")]

    def plan(q, pool=pools["aligned"], extra_out=None):
        srcs = [render.Pooled(pool, pick, (0, WL), 0, render.DryStream(up, ids, ids, q))]
        p = R.plan_device(srcs, extra_out or out)
        p.close()

    plan(render.StemLoudness(t[0:1], res[0:2]))                         # accepted
    bad = [
        ("a StemLoudness", (0.0,)),
        ("float64", render.StemLoudness(t[0:1].float())),
        ("1 element", render.StemLoudness(t[0:2])),
        ("CUDA tensor", render.StemLoudness(t[0:1].cpu())),
        ("float64", render.StemLoudness(t[0:1], res[0:2].float())),
        ("2 elements", render.StemLoudness(t[0:1], res[0:3])),
        ("contiguous", render.StemLoudness(t[0:1], res[0:4:2])),
        ("sr", render.StemLoudness(t[0:1], None, 0.0)),
        ("sr", render.StemLoudness(t[0:1], None, -16000.0)),
        ("meets", render.StemLoudness(t[0:1], t[0:2])),                  # the result is the target
    ]
    for what, q in bad:
        with pytest.raises(ValueError, match=what):
            plan(q)
    with pytest.raises(ValueError, match="meets"):                      # the result inside an output
        o = torch.empty((2, WL), dtype=torch.float32, device="cuda")
        plan(render.StemLoudness(t[0:1], o.view(torch.float64)[0, :2]), extra_out=[o])
    # two slots writing one result, and slots of different rates
    srcs = [render.Pooled(pools["aligned"], pick, (0, WL), 0,
                          render.DryStream(up, ids, ids, render.StemLoudness(t[k:k + 1], res[0:2]))) for k in range(2)]
    with pytest.raises(ValueError, match="meets"):
        R.plan_device(srcs, out * 2)
    srcs = [render.Pooled(pools["aligned"], pick, (0, WL), 0,
                          render.DryStream(up, ids, ids, render.StemLoudness(t[k:k + 1], None, 16000.0 + k)))
            for k in range(2)]
    with pytest.raises(ValueError, match="one sr"):
        R.plan_device(srcs, [torch.empty((2, WL), device="cuda") for _ in range(2)])
    # a host pool, a tap-form host pool, unequal N, a pool with loudness gains (the existing refusal)
    hp = _host_pool(R, render, cands["aligned"])
    tb = [R.rir_bank(c.h, False, 0, host=True, form="taps") for c in cands["aligned"]]
    tp = R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(cands["aligned"], tb)])
    uneq = speakers(920, n=3, taps=0)
    up_ = R.source_pool([c.src for c in uneq])
    gp = R.source_pool([c.src for c in cands["aligned"]], lufs_targets=[-20.0] * 3, sr=RATE)
    try:
        q = render.StemLoudness(t[0:1])
        for p, what in ((hp, "host pool"), (tp, "host pool"), (up_, "differ in N"), (gp, "loudness gains")):
            with pytest.raises(ValueError, match=what):
                plan(q, pool=p, extra_out=[torch.empty((p.C, WL), device="cuda")])
        # C > 8
        rng = np.random.default_rng(4)
        c9 = [Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 9, 4096)[0], None) for _ in range(2)]
        p9 = R.source_pool([c.src for c in c9])
        try:
            with pytest.raises(ValueError, match="at most 8 channels"):
                plan(q, pool=p9, extra_out=[torch.empty((9, WL), device="cuda")])
        finally:
            p9.close()
    finally:
        for p in (hp, tp, up_, gp):
            p.close()
        for b in tb:
            b.close()


def test_c_abi_refusals(world):
    from sonicsim_b200 import _lib as L
    from sonicsim_b200.SonicSim_audio import gating_block_size, gating_plan
    render, R = _R()
    cands, pools, clips, upools, cpools = world
    up = upools["device"]
    ids = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    lay = torch.full((4, M), -1, dtype=torch.int32, device="cuda")
    pick = torch.zeros(3, dtype=torch.int32, device="cuda")
    t = torch.full((4,), -20.0, dtype=torch.float64, device="cuda")
    res = torch.zeros(8, dtype=torch.float64, device="cuda")
    o = [torch.empty((2, WL), device="cuda") for _ in range(3)]
    srcs = [render.Pooled(pools["aligned"], pick[0:1], (0, WL), 0), render.Pooled(pools["static"], pick[1:2], (0, WL), 0),
            render.Pooled(pools["static"], pick[2:3], (0, WL), 0)]
    items, n, keep = R._device_items(srcs, o)
    strm = (L.SsDryStream * 1)(L.SsDryStream(slot=0, pool=up._h.value, ids_dev=ids.data_ptr(),
                                             offsets_dev=ids.data_ptr(), m=M))
    bgs = (L.SsBgStream * 1)(L.SsBgStream(slot=1, pool=cpools[("int16", "device")]._h.value,
                                          ids_dev=lay[0].data_ptr(), offsets_dev=lay[1].data_ptr(),
                                          heads_dev=lay[2].data_ptr(), counts_dev=lay[3].data_ptr(), m=M))
    block = float(gating_block_size(N, RATE))
    brk, blo, bhi = gating_plan(N, float(RATE), block)

    def G(**kw):
        g = dict(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data, n_e=len(brk) - 1,
                 n_blocks=len(blo), rate=float(RATE), block_size=block)
        g.update(kw)
        return L.SsPostLufs(**g)

    def E(slot=0, g=None, tp=None, rp=0):
        return L.SsStreamLufs(slot=slot, gating=g if g is not None else G(),
                              target_dev=t.data_ptr() if tp is None else tp, result_dev=rp or None)

    def create(entries, items_=None, streams=strm, beds=bgs, count=None):
        arr = (L.SsStreamLufs * len(entries))(*entries) if entries else None
        h = ctypes.c_void_p(12345)
        its, ni = items_ if items_ is not None else (items, n)
        st = R.lib.ss_plan_create_lufs(R.ctx, its, ni, None, 0, None, 0, None, None, 0, None, 0, streams,
                                       1 if streams else 0, beds, 1 if beds else 0, arr,
                                       len(entries) if count is None else count, ctypes.byref(h))
        if st == L.SS_OK:
            R.lib.ss_plan_destroy(h)
            return st
        assert h.value == 12345                                    # *out untouched
        return st

    assert create([E(0, rp=res.data_ptr()), E(1, tp=t.data_ptr() + 8, rp=res.data_ptr() + 16)]) == L.SS_OK
    assert create([]) == L.SS_OK                                   # ss_plan_create_bg
    brk_bad = brk.copy()
    brk_bad[-1] = N + 1
    brk_desc = brk.copy()
    brk_desc[3], brk_desc[4] = brk_desc[4], brk_desc[3]
    bhi_bad = bhi.copy()
    bhi_bad[-1] = len(brk)
    invalid = [
        [E(slot=2)], [E(slot=3)], [E(slot=-1)], [E(0), E(0)],
        [E(g=G(brk=None))], [E(g=G(blk_lo=None))], [E(g=G(n_e=0))], [E(g=G(rate=0.0))], [E(g=G(block_size=NAN))],
        [E(0), E(1, g=G(rate=22050.0))],
        [E(g=G(brk=brk_bad.ctypes.data))], [E(g=G(brk=brk_desc.ctypes.data))], [E(g=G(blk_hi=bhi_bad.ctypes.data))],
        [E(tp=0)], [E(tp=t.data_ptr() + 4)], [E(rp=res.data_ptr() + 4)],
        [E(rp=t.data_ptr())],                                      # the result over the target
        [E(rp=ids.data_ptr())],                                    # ... over the layout
        [E(rp=o[0].data_ptr())],                                   # ... over an output
        [E(0, rp=res.data_ptr()), E(1, tp=t.data_ptr() + 8, rp=res.data_ptr() + 8)],   # two results meet
    ]
    for b in invalid:
        assert create(b) == L.SS_ERR_INVALID, b
    assert create([E()], count=-1) == L.SS_ERR_INVALID
    h = ctypes.c_void_p()
    assert R.lib.ss_plan_create_lufs(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0, strm, 1, bgs, 1,
                                     None, 1, ctypes.byref(h)) == L.SS_ERR_INVALID and not h.value
    # unsupported: a host pool, a tap-form host pool, unequal N, C > 8
    hp = _host_pool(R, render, cands["aligned"])
    tb = [R.rir_bank(c.h, False, 0, host=True, form="taps") for c in cands["aligned"]]
    tp = R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(cands["aligned"], tb)])
    uneq = R.source_pool([c.src for c in speakers(921, n=3, taps=0)])
    rng = np.random.default_rng(4)
    c9 = [Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 9, 4096)[0], None) for _ in range(2)]
    p9 = R.source_pool([c.src for c in c9])
    try:
        for p in (hp, tp, uneq, p9):
            wl = min(WL, p.n_min)
            o2 = [torch.empty((p.C, wl), device="cuda")]
            its = R._device_items([render.Pooled(p, pick[0:1], (0, wl), 0)], o2)
            assert create([E()], items_=its[:2], beds=None) == L.SS_ERR_UNSUPPORTED, p
    finally:
        for p in (hp, tp, uneq, p9):
            p.close()
        for b in tb:
            b.close()
