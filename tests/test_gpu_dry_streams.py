"""Dry streams (render.DryStream; ss_plan_create_stream) through the real kernels.  Every plan is run twice on the same
picks, starts, variates, SIRs and SNRs: once with stream slots, whose layouts (ids, offsets) change at every run with no
re-plan, and once with the same slots dry-picking, from a 16-bit dry pool, the streams those layouts lay out, assembled
on the host to the slot pool's longest N.  Checked, bit for bit:
  1. stems and direct stems over the aligned k_render_fast pool (direct sets), a grid pool (K = 3), a mixed-length
     long-RIR pool (K = 2..4) and static noise, for device and host source pools crossed with device and host utterance
     pools, over several runs, one of them on a side stream behind queued work; and against render_device of the
     picked candidate with the assembled stream;
  2. training steps with start draws over two stream speakers, mixtures per channel and mono, speakers_out, rms_db,
     dereverberation targets, drawn starts and `used`;
  3. stream slots of a host pool of tap-form banks (the plan's k_stage then stages taps and stream samples);
  4. an utterance pool closed under a live plan: the plan keeps its bits, the memory returns with the plan;
  5. invalid layout entries are skipped, with bit 5 raising ValueError from check_device_errors;
  6. refusals in Python and through the C ABI, with no plan created, slot pools beyond 2^23 samples included."""
import ctypes
import gc

import numpy as np
import pytest
import torch

from gpu_plumbing import _R
from pool_worlds import _host_pool, longs, moving, noises, reference, speakers

pytestmark = pytest.mark.gpu

TAPS = 40
NAN = float("nan")
RATE = 16000
SLEEP = int(5e8)
M = 24


def utterance_pool_signals(seed, n, lo, hi):
    """n int16 utterances of lo..hi samples: speech-like bursts at random levels, some with N % 4 != 0."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        k = int(rng.integers(lo, hi + 1))
        v = np.cumsum(rng.standard_normal(k)) * 0.02 + rng.standard_normal(k)
        v *= rng.uniform(0.05, 0.9) / max(1e-9, np.abs(v).max())
        out.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
    return out


def walk(ids, offs, lengths):
    kept, bad, end = [], False, 0
    for i, o in zip(ids, offs):
        if i < 0:
            continue
        if i >= len(lengths) or o < 0 or o < end:
            bad = True
            continue
        kept.append((int(i), int(o)))
        end = o + lengths[i]
    return kept, bad


def assemble(ids, offs, utts, cut):
    k = np.zeros(cut, np.int16)
    for i, o in walk(ids, offs, [u.size for u in utts])[0]:
        if o < cut:
            n = min(utts[i].size, cut - o)
            k[o:o + n] = utts[i][:n]
    return k


def random_layouts(rng, k, n, lengths, cut, invalid=False):
    """k layouts of M entries: utterances with gaps of 0..1.5 s from a random start, a few empty entries, the last
    placements reaching past cut; with `invalid`, some entries invalid."""
    ids, offs = np.full((k, M), -1, np.int32), np.full((k, M), -1, np.int32)
    for j in range(k):
        pos, e = int(rng.integers(-RATE, RATE)), 0
        while e < M and pos < cut + RATE:
            if rng.random() < 0.1:
                e += 1
                continue
            i = int(rng.integers(0, n))
            o = max(0, pos)
            ids[j, e], offs[j, e] = i, o
            if invalid and rng.random() < 0.15:
                ids[j, e], offs[j, e] = [(n, o), (i, -3), (i, max(0, o - 1 - int(rng.integers(0, 500))))][
                    int(rng.integers(0, 3))]
                if offs[j, e] >= o:
                    offs[j, e] = o - 1 if o > 0 else -1
            pos = o + lengths[i] + int(rng.integers(0, int(1.5 * RATE)))
            e += 1
    return ids, offs


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    kinds = {"aligned": (speakers(701, n=4, taps=TAPS), TAPS), "grid": (longs(702), 0),
             "mixedK": (moving(703, [5000, 9000, 13000, 6000]), 0), "noise": (noises(704, n=3), 0)}
    out = {}
    for kind, (cands, taps) in kinds.items():
        out[kind] = (cands, taps, {"device": R.source_pool([c.src for c in cands]),
                                   "host": _host_pool(R, render, cands, taps)})
    utts = utterance_pool_signals(705, 9, 1, int(1.2 * RATE))
    utts[3] = utts[3][:1]                                          # a one-sample utterance
    upools = {res: R.dry_pool(utts, levels=True, host=res == "host", dtype="int16") for res in ("device", "host")}
    yield out, utts, upools
    for _, _, pools in out.values():
        for p in pools.values():
            p.close()
    for p in upools.values():
        p.close()


class Arms:
    """k pooled slots over one pool: stream slots (ids, offs rows) and their twins dry-picking the assembled streams."""

    def __init__(self, R, render, pool, upool, cands, wl, taps, k=4):
        self.k, self.wl, self.taps, self.cands = k, wl, taps, cands
        d = "cuda"
        self.picks = torch.zeros(k, dtype=torch.int32, device=d)
        self.starts = torch.zeros(k, dtype=torch.int32, device=d)
        self.ids = torch.full((k, M), -1, dtype=torch.int32, device=d)
        self.offs = torch.full((k, M), -1, dtype=torch.int32, device=d)
        self.dpicks = torch.arange(k, dtype=torch.int32, device=d)
        C = cands[0].C
        self.outs = [torch.empty((C, wl), device=d) for _ in range(2 * k)]
        self.douts = [torch.empty((C, wl), device=d) for _ in range(2 * k)] if taps else None
        self.srcs = [render.Pooled(pool, self.picks[j], (self.starts[j], wl), taps,
                                   render.DryStream(upool, self.ids[j], self.offs[j])) for j in range(k)]
        self.plan = R.plan_device(self.srcs, self.outs[:k], direct_outs=self.douts[:k] if taps else None)
        self.pool, self.render, self.R = pool, render, R

    def oracle(self, streams, host):
        """The twin plan over a 16-bit pool of this run's assembled streams (the oracle is re-planned every run)."""
        apool = self.R.dry_pool(streams, host=host, dtype="int16")
        srcs = [self.render.Pooled(self.pool, self.picks[j], (self.starts[j], self.wl), self.taps,
                                   self.render.DryPick(apool, self.dpicks[j])) for j in range(self.k)]
        plan = self.R.plan_device(srcs, self.outs[self.k:], direct_outs=self.douts[self.k:] if self.taps else None)
        return apool, plan

    def results(self):
        return self.outs + (self.douts or [])


@pytest.mark.parametrize("u_resident", ["device", "host"])
@pytest.mark.parametrize("src_resident", ["device", "host"])
@pytest.mark.parametrize("kind", ["aligned", "grid", "mixedK", "noise"])
def test_stems_equal_the_assembled_pick(world, kind, src_resident, u_resident):
    render, R = _R()
    out, utts, upools = world
    cands, taps, pools = out[kind]
    upool, lengths = upools[u_resident], [u.size for u in utts]
    cut, n_min = max(c.N for c in cands), min(c.N for c in cands)
    wl = min(9000, n_min - 1) if kind != "noise" else 20000
    A = Arms(R, render, pools[src_resident], upool, cands, wl, taps)
    rng = np.random.default_rng(["aligned", "grid", "mixedK", "noise"].index(kind) * 4 + 2 * (src_resident == "host") +
                                (u_resident == "host"))
    side = torch.cuda.Stream()
    try:
        for run in range(4):
            ids, offs = random_layouts(rng, A.k, len(utts), lengths, cut)
            if run == 0:                                  # a stream wholly of gaps, and one of the longest utterances
                ids[0], offs[0] = -1, 0
                ids[1], offs[1] = -1, 0
                ids[1, :3], offs[1, :3] = [0, 1, 2], [0, lengths[0], lengths[0] + lengths[1]]
            A.ids.copy_(torch.from_numpy(ids))
            A.offs.copy_(torch.from_numpy(offs))
            A.picks.copy_(torch.from_numpy(rng.integers(0, len(cands), A.k).astype(np.int32)))
            A.starts.copy_(torch.from_numpy(rng.integers(0, n_min - wl + 1, A.k).astype(np.int32)))
            if run == 0:
                A.picks.fill_(int(np.argmax([c.N for c in cands])))
                A.starts.copy_(torch.tensor([0, cut - wl, cut - wl, 0], dtype=torch.int32))
            streams = [assemble(ids[j], offs[j], utts, cut) for j in range(A.k)]
            apool, oplan = A.oracle(streams, u_resident == "host")
            for t in A.results():
                t.fill_(NAN)
            if run == 2:                                  # on a side stream behind queued work
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
            k = A.k
            for j in range(k):
                assert torch.isfinite(A.outs[j]).all() and torch.equal(A.outs[j], A.outs[k + j]), (kind, run, j)
                if taps:
                    assert torch.equal(A.douts[j], A.douts[k + j]), (kind, run, j)
            if run == 1:                                  # and against render_device with the assembled stream
                for j in range(k):
                    c = cands[int(A.picks[j])]
                    x = torch.from_numpy(streams[j].astype(np.float32) / np.float32(32768)).cuda()
                    ref, dref = reference(c, x, int(A.starts[j]), wl, taps)
                    assert torch.equal(A.outs[j], ref), (kind, j)
                    if taps:
                        assert torch.equal(A.douts[j], dref), (kind, j)
            oplan.close()
            apool.close()
        assert A.plan.is_graph()
    finally:
        A.plan.close()


def run_twins(A, rng, utts, cut, u_host, runs=3):
    """Runs A's stream plan and its assembled-pick twin on fresh layouts, picks and starts; asserts equal bits."""
    lengths, n_min = [u.size for u in utts], min(c.N for c in A.cands)
    for run in range(runs):
        ids, offs = random_layouts(rng, A.k, len(utts), lengths, cut)
        A.ids.copy_(torch.from_numpy(ids))
        A.offs.copy_(torch.from_numpy(offs))
        A.picks.copy_(torch.from_numpy(rng.integers(0, len(A.cands), A.k).astype(np.int32)))
        A.starts.copy_(torch.from_numpy(rng.integers(0, n_min - A.wl + 1, A.k).astype(np.int32)))
        apool, oplan = A.oracle([assemble(ids[j], offs[j], utts, cut) for j in range(A.k)], u_host)
        for t in A.results():
            t.fill_(NAN)
        A.plan.run()
        oplan.run()
        torch.cuda.synchronize()
        A.R.check_device_errors()
        for x, y in zip(A.outs[:A.k] + (A.douts or [])[:A.k], A.outs[A.k:] + (A.douts or [])[A.k:]):
            assert torch.isfinite(x).all() and torch.equal(x, y), run
        oplan.close()
        apool.close()


@pytest.mark.parametrize("u_resident", ["device", "host"])
def test_stream_slots_of_a_tap_form_host_pool(world, u_resident):
    """Stream slots of a host pool of tap-form banks (k_stage<true, true, true>, then the plan's transform launch)
    against their assembled-pick twins (k_stage<true, true>), direct stems included."""
    render, R = _R()
    out, utts, upools = world
    cands, taps, _ = out["aligned"]
    banks = [R.rir_bank(c.h, False, TAPS, host=True, form="taps") for c in cands]
    pool = R.source_pool([render.MovingSource(c.x, b, c.b, c.b) for c, b in zip(cands, banks)])
    A = Arms(R, render, pool, upools[u_resident], cands, 9000, TAPS)
    try:
        run_twins(A, np.random.default_rng(31 + (u_resident == "host")), utts, max(c.N for c in cands),
                  u_resident == "host")
    finally:
        A.plan.close()
        pool.close()
        for b in banks:
            b.close()


def test_utterance_pool_closed_under_a_live_plan(world):
    """close() of an utterance pool that a live stream plan uses: new plans refuse it at once, the plan keeps running
    with its bits (fresh allocations meanwhile would reuse the pool's memory had it been freed), and the pool is
    destroyed only when the plan is closed.  (The pool's handle tells: device-wide free memory also moves with other
    processes on a shared GPU.)"""
    render, R = _R()
    out, _, _ = world
    cands, taps, pools = out["aligned"]
    rng = np.random.default_rng(41)
    utts = utterance_pool_signals(42, 80, 20 * RATE, 30 * RATE)
    cut = max(c.N for c in cands)
    up = R.dry_pool(utts, levels=True, dtype="int16")
    assert up.nbytes >= 50e6
    A = Arms(R, render, pools["device"], up, cands, 9000, taps)
    try:
        run_twins(A, rng, utts, cut, False, runs=1)        # the plan's bits against the assembled picks
        before = [t.clone() for t in A.results()[:A.k]] + [t.clone() for t in (A.douts or [])[:A.k]]
        up.close()
        assert up.closed and up._h.value and up._plans == 1   # refused to new plans, held by the live one
        with pytest.raises(ValueError, match="is closed"):
            R.plan_device([render.Pooled(pools["device"], A.picks[0], (A.starts[0], 9000), taps,
                                         render.DryStream(up, A.ids[0], A.offs[0]))], [torch.empty((2, 9000),
                                                                                                    device="cuda")])
        junk = [torch.full((1 << 24,), 7.0, device="cuda") for _ in range(4)]
        for _ in range(2):
            for t in A.results():
                t.fill_(NAN)
            A.plan.run()
            torch.cuda.synchronize()
            after = [t for t in A.results()[:A.k]] + [t for t in (A.douts or [])[:A.k]]
            for x, y in zip(before, after):
                assert torch.equal(x, y)
        R.check_device_errors()
        del junk
        A.plan.close()
        gc.collect()
        assert not up._h.value and up._plans == 0           # destroyed with the last plan that used it
    finally:
        A.plan.close()
        up.close()


# ------------------------------------------------------------------------------------------- 2. draws and mixtures
LEN = RATE


class Step:
    """B examples: two speakers (stream slots, or their assembled-pick twins), a pooled noise without a dry signal; one
    CropDraw over both speakers, one mixture per channel with dereverberation targets and one mono."""

    def __init__(self, R, render, sp, npool, B, dry_of, thr=-35.0, tries=37):
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
            srcs += [render.Pooled(sp, self.picks[b, 0], w, TAPS, dry_of(b, 0)),
                     render.Pooled(sp, self.picks[b, 1], w, TAPS, dry_of(b, 1)),
                     render.Pooled(npool, self.picks[b, 2], w)]
            draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], self.u[b], self.used[b], thr))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mix[b],
                                        self.spo[b], self.rms[b], direct_out=self.tgt[b]))
            mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mmix[b],
                                        self.mspo[b], self.mrms[b], mono=True))
        self.plan = R.plan_device(srcs, self.outs, direct_outs=self.douts, mixtures=mixes, draws=draws)

    def results(self):
        for t in self.outs + [d for d in self.douts if d is not None] + [self.mix, self.spo, self.tgt, self.rms,
                                                                          self.mmix, self.mspo, self.mrms]:
            yield t
        yield self.starts
        yield self.used

    def clear(self):
        for t in self.outs + [d for d in self.douts if d is not None] + [self.mix, self.spo, self.tgt, self.rms,
                                                                          self.mmix, self.mspo, self.mrms]:
            t.fill_(NAN)
        self.starts.fill_(-1)
        self.used.fill_(-7)


@pytest.mark.parametrize("u_resident", ["device", "host"])
@pytest.mark.parametrize("src_resident", ["device", "host"])
def test_draws_mixtures_and_targets_equal_the_assembled_pick(world, src_resident, u_resident):
    render, R = _R()
    out, utts, upools = world
    spk, _, spools = out["aligned"]
    noi, _, npools = out["noise"]
    upool, lengths = upools[u_resident], [u.size for u in utts]
    cut = max(c.N for c in spk)
    B = 8
    ids = torch.full((B, 2, M), -1, dtype=torch.int32, device="cuda")
    offs = torch.full((B, 2, M), -1, dtype=torch.int32, device="cuda")
    S = Step(R, render, spools[src_resident], npools[src_resident], B,
             lambda b, s: render.DryStream(upool, ids[b, s], offs[b, s]))
    rng = np.random.default_rng(77 + len(src_resident) + 3 * len(u_resident))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7)
    outcomes = set()
    try:
        for run in range(4):
            lay = [random_layouts(rng, 2, len(utts), lengths, cut) for _ in range(B)]
            ids.copy_(torch.from_numpy(np.stack([a for a, _ in lay])))
            offs.copy_(torch.from_numpy(np.stack([o for _, o in lay])))
            streams = [assemble(lay[b][0][s], lay[b][1][s], utts, cut) for b in range(B) for s in range(2)]
            apool = R.dry_pool(streams, levels=True, host=u_resident == "host", dtype="int16")
            dp = torch.arange(2 * B, dtype=torch.int32, device="cuda").reshape(B, 2)
            T = Step(R, render, spools[src_resident], npools[src_resident], B,
                     lambda b, s: render.DryPick(apool, dp[b, s]))
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
            for j, (x, y) in enumerate(zip(S.results(), T.results())):
                assert torch.equal(x, y), (run, j)
            outcomes |= {"first" if v == 1 else "later" if v > 1 else "none" for v in S.used.cpu().numpy()}
            T.plan.close()
            apool.close()
        assert "later" in outcomes and "first" in outcomes, outcomes     # crops in gaps were rejected
    finally:
        S.plan.close()


# --------------------------------------------------------------------------------------------------- 3. bit 5
def test_invalid_entries_are_skipped_and_reported(world):
    render, R = _R()
    out, utts, upools = world
    cands, taps, pools = out["aligned"]
    lengths = [u.size for u in utts]
    cut, n_min = max(c.N for c in cands), min(c.N for c in cands)
    A = Arms(R, render, pools["device"], upools["host"], cands, 8000, taps)
    rng = np.random.default_rng(55)
    try:
        ids, offs = random_layouts(rng, A.k, len(utts), lengths, cut, invalid=True)
        assert any(walk(ids[j], offs[j], lengths)[1] for j in range(A.k))
        A.ids.copy_(torch.from_numpy(ids))
        A.offs.copy_(torch.from_numpy(offs))
        A.starts.copy_(torch.from_numpy(rng.integers(0, n_min - 8000 + 1, A.k).astype(np.int32)))
        apool, oplan = A.oracle([assemble(ids[j], offs[j], utts, cut) for j in range(A.k)], False)
        A.plan.run()
        oplan.run()
        with pytest.raises(ValueError, match="DryStream"):
            R.check_device_errors()
        for j in range(A.k):
            assert torch.equal(A.outs[j], A.outs[A.k + j]) and torch.equal(A.douts[j], A.douts[A.k + j])
        # valid layouts again: no report
        ids, offs = random_layouts(rng, A.k, len(utts), lengths, cut)
        A.ids.copy_(torch.from_numpy(ids))
        A.offs.copy_(torch.from_numpy(offs))
        A.plan.run()
        R.check_device_errors()
        oplan.close()
        apool.close()
    finally:
        A.plan.close()


# ------------------------------------------------------------------------------------------------- 4. refusals
def test_python_refusals(world):
    render, R = _R()
    out, utts, upools = world
    cands, taps, pools = out["aligned"]
    pool, up = pools["device"], upools["device"]
    ids = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    offs = torch.zeros(M, dtype=torch.int32, device="cuda")
    pick, start = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    o = [torch.empty((2, 4000), device="cuda")]

    def plan(d, p=pool, draws=None):
        return R.plan_device([render.Pooled(p, pick, (start, 4000), 0, d)], o, draws=draws)

    fl = R.dry_pool([torch.zeros(cut_len(cands), device="cuda")])
    nolev = R.dry_pool([u for u in utts], dtype="int16")
    gp = R.source_pool([c.src for c in cands], lufs_targets=[-20.0] * len(cands))
    try:
        for d, p, match in [
            (render.DryStream(fl, ids, offs), pool, "16-bit"),
            (render.DryStream(up, ids, offs), gp, "loudness gains"),
            (render.DryStream(up, ids.long(), offs), pool, "int32"),
            (render.DryStream(up, ids, offs[:5]), pool, "shape"),
            (render.DryStream(up, ids.cpu(), offs), pool, "CUDA"),
            (render.DryStream(up, torch.full((129,), -1, dtype=torch.int32, device="cuda"),
                              torch.zeros(129, dtype=torch.int32, device="cuda")), pool, "1 to 128"),
            (render.DryStream(up, ids[:0], offs[:0]), pool, "1 to 128"),
            (render.DryStream(up, ids.reshape(4, 6), offs), pool, "shape"),
            (render.DryStream("pool", ids, offs), pool, "DryPool"),
        ]:
            with pytest.raises(ValueError, match=match):
                plan(d, p)
        u = torch.rand(5, dtype=torch.float64, device="cuda")
        with pytest.raises(ValueError, match="level tables"):
            plan(render.DryStream(nolev, ids, offs), draws=[render.CropDraw(start, [0], u)])
        with pytest.raises(ValueError, match="not a pooled slot"):
            c = cands[0]
            R.plan_device([c.src._replace(window=(0, 4000), dry=render.DryStream(up, ids, offs))], o)
    finally:
        fl.close()
        nolev.close()
        gp.close()


def cut_len(cands):
    return max(c.N for c in cands)


def test_c_abi_refusals(world):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    out, utts, upools = world
    cands, taps, pools = out["aligned"]
    pool, up = pools["device"], upools["device"]
    ids = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    offs = torch.zeros(M + 1, dtype=torch.int32, device="cuda")
    pick = torch.zeros(2, dtype=torch.int32, device="cuda")
    o = [torch.empty((2, 4000), device="cuda") for _ in range(2)]
    srcs = [render.Pooled(pool, pick[j:j + 1], (0, 4000), 0) for j in range(2)]
    items, n, keep = R._device_items(srcs, o)
    fl = R.dry_pool([torch.zeros(cut_len(cands), device="cuda")])
    try:
        def create(streams, picks=None, mixes=None, draws=None, items_=None):
            arr = (L.SsDryStream * len(streams))(*streams) if streams else None
            pk = (L.SsDryPick * len(picks))(*picks) if picks else None
            h = ctypes.c_void_p()
            its, ni = items_ if items_ is not None else (items, n)
            st = R.lib.ss_plan_create_stream(R.ctx, its, ni, mixes, len(mixes) if mixes else 0, draws,
                                             len(draws) if draws else 0, pk,
                                             None, len(picks) if picks else 0, None, 0, arr,
                                             len(streams) if streams else 0, ctypes.byref(h))
            if h.value:
                R.lib.ss_plan_destroy(h)
            return st, h.value

        def S(slot=0, pool_h=None, i=None, f=None, m=M):
            return L.SsDryStream(slot=slot, pool=pool_h if pool_h is not None else up._h.value,
                                 ids_dev=ids.data_ptr() if i is None else i,
                                 offsets_dev=offs.data_ptr() if f is None else f, m=m)

        assert create([S()])[0] == L.SS_OK
        assert create([])[0] == L.SS_OK                   # no streams: ss_plan_create_target
        bad = [
            [S(slot=2)], [S(slot=-1)], [S(), S()], [S(m=0)], [S(m=129)], [S(pool_h=fl._h.value)],
            [S(i=0)], [S(f=0)], [S(i=ids.data_ptr() + 2)], [S(f=offs.data_ptr() + 1)],
        ]
        for b in bad:
            assert create(b)[0] == L.SS_ERR_INVALID, b
        # a slot named by a stream and a dry pick
        apool = R.dry_pool([torch.zeros(cut_len(cands), device="cuda")])
        assert create([S()], picks=[L.SsDryPick(slot=0, pool=apool._h.value, pick_dev=pick.data_ptr())])[0] == \
            L.SS_ERR_INVALID
        apool.close()
        # a mixture writing over the layout
        sirs = torch.zeros(1, device="cuda")
        mx = (L.SsPlanMix * 1)()
        mx[0].speakers[0], mx[0].noises[0], mx[0].S, mx[0].M = 0, 1, 1, 1
        mx[0].snr, mx[0].mix = sirs.data_ptr(), ids.data_ptr()
        assert create([S()], mixes=mx)[0] == L.SS_ERR_INVALID
        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_stream(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0, None, 1,
                                           ctypes.byref(h)) == L.SS_ERR_INVALID and not h.value
        # a NULL dry pool, and one of another context
        assert create([S(pool_h=0)])[0] == L.SS_ERR_INVALID
        ctx2 = ctypes.c_void_p()
        L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
        R2 = render.Renderer(R.device)
        R2.ctx = ctx2
        foreign = R2.dry_pool(utts, levels=True, dtype="int16")
        try:
            assert create([S(pool_h=foreign._h.value)])[0] == L.SS_ERR_INVALID
        finally:
            foreign.close()
            R2.lib.ss_destroy(ctx2)
        # a slot that is not pooled, and a slot of a pool with loudness gains
        gp = R.source_pool([c.src for c in cands], lufs_targets=[-20.0] * len(cands))
        try:
            items2, n2, keep2 = R._device_items([cands[0].src._replace(window=(0, 4000)),
                                                 render.Pooled(gp, pick[1:2], (0, 4000), 0)], o)
            assert create([S(slot=1)], items_=(items2, n2))[0] == L.SS_ERR_INVALID
            assert create([S(slot=0)], items_=(items2, n2))[0] == L.SS_ERR_INVALID
        finally:
            gp.close()
        # a draw speaker whose stream's dry pool has no level tables (with tables: accepted)
        start = torch.zeros(1, dtype=torch.int32, device="cuda")
        u = torch.rand(5, dtype=torch.float64, device="cuda")
        items3, n3, keep3 = R._device_items([render.Pooled(pool, pick[0:1], (start, 4000), 0)], o[:1])
        dr = (L.SsPlanDraw * 1)()
        dr[0].start, dr[0].u, dr[0].S, dr[0].tries, dr[0].threshold_db = start.data_ptr(), u.data_ptr(), 1, 5, -40.0
        dr[0].speakers[0] = 0
        nolev = R.dry_pool(utts, dtype="int16")
        try:
            assert create([S(pool_h=nolev._h.value)], draws=dr, items_=(items3, n3))[0] == L.SS_ERR_INVALID
            assert create([S()], draws=dr, items_=(items3, n3))[0] == L.SS_OK
        finally:
            nolev.close()
    finally:
        fl.close()


def test_slot_pools_beyond_2_pow_23_samples_are_unsupported(world):
    """A stream slot over a pool whose longest candidate has 2^23 + 1 samples: SS_ERR_UNSUPPORTED through the C ABI, a
    ValueError in Python; 2^23 samples are accepted."""
    from sonicsim_b200 import _lib as L
    render, R = _R()
    _, utts, upools = world
    up = upools["device"]
    rng = np.random.default_rng(9)
    h = (rng.standard_normal((1, 64)) * 0.1).astype(np.float32)
    ids = torch.full((M,), -1, dtype=torch.int32, device="cuda")
    offs = torch.zeros(M, dtype=torch.int32, device="cuda")
    pick = torch.zeros(1, dtype=torch.int32, device="cuda")
    o = [torch.empty((1, 4000), device="cuda")]
    for N, ok in ((1 << 23, True), ((1 << 23) + 1, False)):
        bank = R.rir_bank(torch.from_numpy(h).cuda())
        pool = R.source_pool([render.StaticSource(torch.zeros(N, device="cuda"), bank)])
        try:
            srcs = [render.Pooled(pool, pick, (0, 4000), 0, render.DryStream(up, ids, offs))]
            if ok:
                R.plan_device(srcs, o).close()
            else:
                with pytest.raises(ValueError, match="2\\^23"):
                    R.plan_device(srcs, o)
            items, n, keep = R._device_items([render.Pooled(pool, pick, (0, 4000), 0)], o)
            st = L.SsDryStream(slot=0, pool=up._h.value, ids_dev=ids.data_ptr(), offsets_dev=offs.data_ptr(), m=M)
            hp = ctypes.c_void_p()
            rc = R.lib.ss_plan_create_stream(R.ctx, items, n, None, 0, None, 0, None, None, 0, None, 0,
                                             (L.SsDryStream * 1)(st), 1, ctypes.byref(hp))
            if hp.value:
                R.lib.ss_plan_destroy(hp)
            assert rc == (L.SS_OK if ok else L.SS_ERR_UNSUPPORTED), (N, rc)
        finally:
            pool.close()
            bank.close()
