"""Background streams (render.BackgroundStream) at training scale against float64.  A pinned host float32 clip pool of
1000 clips of 10 to 60 s (one in eight of 60 s, DnR's resampled length; 1.9 GB, within the pinned budget of a scale
test) serves a 64-example training plan: two speakers over a device pool of moving candidates with 4 s crops, a noise
bed and a music bed over a device pool of static 50 s and 60 s candidates, and a mixture per example.  At every step
dry.background_audio_layouts refreshes both beds' layouts on the device (60 s beds, the noise bed selecting on
44.1 kHz lengths as SonicSet's JSONs list them), with no re-plan.  At every step:
  - every layout is valid and the plan reports no invalid entry;
  - sampled bed stems pass the float64 render of their picked candidate with the assembled bed (ScaleCand.check);
  - the mixtures are finite."""
import numpy as np
import pytest
import torch

from gpu_plumbing import _R, pmap
from oracle import sonicsim_oracle as so
from pool_worlds import PINNED_MAX, DevPool, ScaleCand, a_aligned

from sonicsim_b200 import dry

pytestmark = pytest.mark.gpu

RATE = 16000
WL = 4 * RATE
B = 64
M = 16
N_CLIP = 1000


def walk(ids, offs, heads, counts, lengths):
    kept, end = [], 0
    for i, o, h, c in zip(ids, offs, heads, counts):
        if i < 0:
            continue
        assert 0 <= i < len(lengths) and o >= end and h >= 0 and c >= 1 and h + c <= lengths[i]
        kept.append((i, o, h, c))
        end = o + c
    return kept


def assemble(lay, clips, cut):
    k = np.zeros(cut, np.float32)
    for i, o, h, c in walk(*lay, [x.size for x in clips]):
        if o < cut:
            n = min(c, cut - o)
            k[o:o + n] = clips[i][h:h + n]
    return k


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    rng = np.random.default_rng(2027)
    base = (rng.standard_normal(1 << 26) * 0.2).astype(np.float32)
    lengths = np.where(rng.random(N_CLIP) < 0.125, 60 * RATE, rng.integers(10 * RATE, 40 * RATE + 1, N_CLIP))
    starts = rng.integers(0, (1 << 26) - lengths)
    gains = rng.uniform(0.05, 1.0, N_CLIP).astype(np.float32)
    clips = [base[a:a + n] * g for a, n, g in zip(starts, lengths, gains)]
    cpool = R.dry_pool(clips, host=True)
    assert cpool.host_nbytes <= PINNED_MAX, cpool.host_nbytes
    spk = DevPool(a_aligned(rng))
    bed = DevPool([ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 4096), None)
                   for N in (50 * RATE + 7, 60 * RATE)])
    yield render, R, clips, cpool, spk, bed
    cpool.close()
    spk.pool.close()
    bed.pool.close()


def test_training_steps_of_fresh_beds(world):
    render, R, clips, cpool, spk, bed = world
    d = "cuda"
    lengths = torch.tensor([c.size for c in clips], dtype=torch.int64, device=d)
    native = (lengths * 441) // 160                     # the lengths a SonicSet JSON lists at 44.1 kHz
    lay = torch.full((4, B, 2, M), -1, dtype=torch.int32, device=d)
    picks = torch.zeros((B, 4), dtype=torch.int32, device=d)
    starts = torch.zeros(B, dtype=torch.int32, device=d)
    sirs, snr = torch.zeros((B, 1), device=d), torch.zeros(B, device=d)
    outs = [torch.empty((2, WL), device=d) for _ in range(4 * B)]
    mix, spo = torch.empty((B, 2, WL), device=d), torch.empty((B, 2, 2, WL), device=d)
    rms = torch.empty((B, 2), device=d)
    srcs, mixes = [], []
    for b in range(B):
        w = (starts[b], WL)
        srcs += [render.Pooled(spk.pool, picks[b, 0], w), render.Pooled(spk.pool, picks[b, 1], w)]
        srcs += [render.Pooled(bed.pool, picks[b, 2 + q], w, 0,
                               render.BackgroundStream(cpool, *[lay[f, b, q] for f in range(4)])) for q in range(2)]
        mixes.append(render.Mixture([4 * b, 4 * b + 1], [4 * b + 2, 4 * b + 3], sirs[b], snr[b], mix[b], spo[b],
                                    rms[b]))
    plan = R.plan_device(srcs, outs, mixtures=mixes)
    cut = bed.n_max
    n_min = min(min(c.N for c in spk.cands), min(c.N for c in bed.cands))
    gen = torch.Generator(device=d)
    gen.manual_seed(13)
    rng = np.random.default_rng(14)
    trimmed = placed = 0
    try:
        for step in range(3):
            for q, sel in ((0, native), (1, None)):
                for f, v in enumerate(dry.background_audio_layouts(lengths, 60 * RATE, M, B, generator=gen,
                                                                   select_lengths=sel)):
                    lay[f, :, q].copy_(v)
            picks[:, :2].copy_(torch.randint(0, len(spk.cands), (B, 2), generator=gen, device=d, dtype=torch.int32))
            picks[:, 2:].copy_(torch.randint(0, len(bed.cands), (B, 2), generator=gen, device=d, dtype=torch.int32))
            starts.copy_(torch.randint(0, n_min - WL + 1, (B,), generator=gen, device=d, dtype=torch.int32))
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(5, 20, generator=gen)
            for t in outs:
                t.fill_(float("nan"))
            plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            assert torch.isfinite(mix).all()
            L, P, S = (t.cpu().numpy() for t in (lay, picks, starts))
            for b in range(B):
                for q in range(2):
                    kept = walk(*L[:, b, q], [c.size for c in clips])
                    placed += len(kept)
                    trimmed += sum(1 for i, o, h, c in kept if h > 0 or c < clips[i].size)
            jobs = []
            for b in rng.choice(B, 6, replace=False):
                for q in range(2):
                    c = bed.cands[P[b, 2 + q]]
                    x = assemble(L[:, b, q], clips, cut)[:c.N]
                    jobs.append((ScaleCand(x, c.h, None), outs[4 * b + 2 + q].cpu().numpy(), int(S[b]),
                                 "step %d example %d bed %d" % (step, b, q)))
            pmap(lambda j: j[0].check(j[1], j[2], WL, key="bed", label=j[3]), jobs)
        assert placed > 4 * B and trimmed > B // 2      # beds of one or more clips, many with a trimmed end clip
    finally:
        plan.close()
