"""Dry streams (render.DryStream) at training scale against float64.  A 16-bit utterance pool of 20000 synthetic
utterances of 1 to 35 s (about 11.5 GB of int16 samples, with sparse level tables) serves a 64-example training plan:
two stream speakers per example over a device pool of moving candidates with 4 s crops drawn under the silence rule, a
pooled static noise, and a mixture per example.  Over several steps the layouts are refreshed on the device by
dry.long_audio_layouts for 60 s streams (the first step sorting every utterance, the others bounded by
long_audio_max_selected), with no re-plan.  At every step:
  - every draw's start and `used` equal draw_reference.draw on the exact level tables (the long-double prefix of the
    float32 squares, exact: DESIGN f13) of the streams the layouts lay out, assembled on the host;
  - sampled speaker stems pass the float64 render of their picked candidate with the assembled stream (ScaleCand.check).
"""
import numpy as np
import pytest
import torch

import draw_reference as dr
from gpu_plumbing import _R, pmap
from oracle import sonicsim_oracle as so
from pool_worlds import DevPool, ScaleCand, a_aligned
from render_reference import graded_dry

from sonicsim_b200 import dry

pytestmark = pytest.mark.gpu

RATE = 16000
WL = 4 * RATE
B = 64
M = 32
THR = -40.0
TRIES = 101


def exact_table(k):
    v = k.astype(np.float32) / np.float32(32768)
    return dr.level_table(v[None], True, np.longdouble).astype(np.float64)


def assemble(ids, offs, utts, cut):
    k = np.zeros(cut, np.int16)
    end = 0
    for i, o in zip(ids, offs):
        if i < 0:
            continue
        assert o >= end                                 # long_audio_layouts never overlaps
        n = utts[i].size
        end = o + n
        if o < cut:
            k[o:min(cut, o + n)] = utts[i][:min(n, cut - o)]
    return k


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    rng = np.random.default_rng(2026)
    base = np.clip(np.round(rng.standard_normal(1 << 26) * 6000), -32768, 32767).astype(np.int16)
    silent = rng.integers(0, (1 << 26) - RATE, 400)     # quiet stretches inside utterances
    for s in silent:
        base[s:s + int(rng.integers(RATE // 4, RATE))] = 0
    lengths = rng.integers(RATE, 35 * RATE + 1, 20000)
    starts = rng.integers(0, (1 << 26) - lengths)
    utts = [base[a:a + n] for a, n in zip(starts, lengths)]
    upool = R.dry_pool(utts, levels=True, dtype="int16")
    spk = DevPool(a_aligned(rng))
    noi = DevPool([ScaleCand(graded_dry(rng, N), so.synth_rirs(rng, 1, 2, 4096), None) for N in (66001, 70002)])
    yield render, R, utts, upool, spk, noi
    upool.close()
    spk.pool.close()
    noi.pool.close()


def test_training_steps_of_fresh_layouts(world):
    render, R, utts, upool, spk, noi = world
    d = "cuda"
    lengths = torch.tensor([u.size for u in utts], dtype=torch.int64, device=d)
    ids = torch.full((B, 2, M), -1, dtype=torch.int32, device=d)
    offs = torch.full((B, 2, M), -1, dtype=torch.int32, device=d)
    picks = torch.zeros((B, 3), dtype=torch.int32, device=d)
    starts = torch.zeros(B, dtype=torch.int32, device=d)
    u = torch.zeros((B, TRIES), dtype=torch.float64, device=d)
    used = torch.zeros(B, dtype=torch.int32, device=d)
    sirs, snr = torch.zeros((B, 1), device=d), torch.zeros(B, device=d)
    outs = [torch.empty((2, WL), device=d) for _ in range(3 * B)]
    mix, spo = torch.empty((B, 2, WL), device=d), torch.empty((B, 2, 2, WL), device=d)
    rms = torch.empty((B, 2), device=d)
    srcs, draws, mixes = [], [], []
    for b in range(B):
        w = (starts[b], WL)
        srcs += [render.Pooled(spk.pool, picks[b, 0], w, 0, render.DryStream(upool, ids[b, 0], offs[b, 0])),
                 render.Pooled(spk.pool, picks[b, 1], w, 0, render.DryStream(upool, ids[b, 1], offs[b, 1])),
                 render.Pooled(noi.pool, picks[b, 2], w)]
        draws.append(render.CropDraw(starts[b], [3 * b, 3 * b + 1], u[b], used[b], THR))
        mixes.append(render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], sirs[b], snr[b], mix[b], spo[b], rms[b]))
    plan = R.plan_device(srcs, outs, mixtures=mixes, draws=draws)
    cut = spk.n_max
    bound = dry.long_audio_max_selected([u.size for u in utts], 60 * RATE)
    assert bound < len(utts)
    gen = torch.Generator(device=d)
    gen.manual_seed(11)
    rng = np.random.default_rng(12)
    outcomes, placed = set(), 0
    try:
        for step in range(3):
            a, o = dry.long_audio_layouts(lengths, 60 * RATE, M, 2 * B, generator=gen,
                                          max_selected=bound if step else None)
            ids.copy_(a.reshape(B, 2, M))
            offs.copy_(o.reshape(B, 2, M))
            picks[:, :2].copy_(torch.randint(0, len(spk.cands), (B, 2), generator=gen, device=d, dtype=torch.int32))
            picks[:, 2].copy_(torch.randint(0, len(noi.cands), (B,), generator=gen, device=d, dtype=torch.int32))
            u.uniform_(generator=gen)
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(5, 20, generator=gen)
            for t in outs:
                t.fill_(float("nan"))
            plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            I, O, P, S, U = (t.cpu().numpy() for t in (ids, offs, picks, starts, used))
            Uv = u.cpu().numpy()
            streams = {}
            for b in range(B):
                for s in range(2):
                    streams[b, s] = assemble(I[b, s], O[b, s], utts, cut)
                    placed += int((I[b, s] >= 0).sum())
                tabs = [exact_table(streams[b, s][:spk.cands[P[b, s]].N]) for s in range(2)]
                reader_N = [spk.cands[P[b, 0]].N, spk.cands[P[b, 1]].N, noi.cands[P[b, 2]].N]
                want = dr.draw(tabs, [WL, WL], reader_N, WL, Uv[b], THR)
                assert (int(S[b]), int(U[b])) == want, (step, b)
                outcomes.add("first" if U[b] == 1 else "later" if U[b] > 1 else "none")
            jobs = []
            for b in rng.choice(B, 6, replace=False):
                for s in range(2):
                    c = spk.cands[P[b, s]]
                    x = streams[b, s][:c.N].astype(np.float32) / np.float32(32768)
                    jobs.append((ScaleCand(x, c.h, c.b), outs[3 * b + s].cpu().numpy(), int(S[b]),
                                 "step %d example %d speaker %d" % (step, b, s)))
            pmap(lambda j: j[0].check(j[1], j[2], WL, key="stream", label=j[3]), jobs)
        assert placed > 2 * B                           # the layouts placed utterances
        assert "later" in outcomes                      # crops in gaps were rejected
    finally:
        plan.close()
