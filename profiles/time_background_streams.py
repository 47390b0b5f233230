"""Background streams in the training step: what it costs to lay out each example's noise and music beds at every run
from clip pools (render.BackgroundStream) instead of dry-picking prebuilt beds (render.DryPick).

Workload: a pool of 32 bench.py configs[1] scenes (64 banked moving speakers, P = 40, C = 6, L = 4096, 30 s) and 32
banked static noise and 32 music candidates in device memory; B = 32 examples per step, each two speakers, a noise
slot and a music slot, one 4 s mono crop per example, SIRs ~ U(-6, 6), SNRs ~ U(10, 20).  The noise slot reads a
float32 device pool of 300 clips of 10 to 60 s, the music slot a 16-bit pinned host pool of 300 clips of 60 s (DnR's
resampled lengths).  Forms, alternating round by round:
(pick) dry picks from 2B prebuilt 30 s beds in a pool of each clip pool's dtype and residency;
(bed)  layouts over the clip pools (m = 16), refreshed by dry.background_audio_layouts (count = B per bed) before
       every step.
Per step: stream time (CUDA events around the step, median), with the layout refresh inside the bed form's step; and
the stream time of background_audio_layouts for 2B rows on its own.  Prints the card and its power limit."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from sonicsim_b200 import dry, render  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, B, SCENES, RATE = 4 * 16000, 32, 32, 16000
N_CLIP, MM = 300, 16
STEPS, ROUNDS = 30, 6


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(7)
    spk_c = [render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in items]

    def statics():
        out = []
        for _ in range(SCENES):
            x = (rng.standard_normal(N) * 0.05).astype(np.float32)
            h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
            out.append(render.StaticSource(to(x), R.rir_bank(to(h))))
        return out

    spk_pool = R.source_pool(spk_c)
    noi_pool, mus_pool = R.source_pool(statics()), R.source_pool(statics())
    noise = [(rng.standard_normal(int(rng.integers(10 * RATE, 60 * RATE))) * 0.1).astype(np.float32)
             for _ in range(N_CLIP)]
    music = [np.clip(np.round(rng.standard_normal(60 * RATE) * 3000), -32768, 32767).astype(np.int16)
             for _ in range(N_CLIP)]
    cp = {"noise": R.dry_pool([to(c) for c in noise]), "music": R.dry_pool(music, host=True, dtype="int16")}
    lens = {"noise": torch.tensor([c.size for c in noise], device=dev),
            "music": torch.tensor([c.size for c in music], device=dev)}
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
    lay = {k: [t.reshape(B, MM) for t in dry.background_audio_layouts(lens[k], N, MM, B, generator=gen)]
           for k in cp}

    def bed(k, row):
        """The bed a layout row lays out, for the prebuilt pools."""
        src = noise if k == "noise" else music
        out = np.zeros(N, src[0].dtype)
        ids, offs, heads, counts = [t[row].cpu().numpy() for t in lay[k]]
        for i, o, h, c in zip(ids, offs, heads, counts):
            if i >= 0 and o < N:
                n = min(c, N - o)
                out[o:o + n] = src[i][h:h + n]
        return out

    pre = {"noise": R.dry_pool([to(bed("noise", j % B)) for j in range(2 * B)]),
           "music": R.dry_pool([bed("music", j % B) for j in range(2 * B)], host=True, dtype="int16")}
    picks = torch.zeros((B, 4), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((B, 2), dtype=torch.int32, device=dev)
    starts = torch.zeros(B, dtype=torch.int32, device=dev)
    sirs, snr = torch.zeros((B, S - 1), device=dev), torch.zeros(B, device=dev)
    outs = [torch.empty((C, CROP), device=dev) for _ in range(4 * B)]
    mix, spo, rms = (torch.empty((B, CROP), device=dev), torch.empty((B, S, CROP), device=dev),
                     torch.empty((B, S), device=dev))

    def plan(form):
        srcs, mixes = [], []
        for b in range(B):
            w = (starts[b], CROP)
            d = [render.BackgroundStream(cp[k], *[t[b] for t in lay[k]]) if form == "bed" else
                 render.DryPick(pre[k], dpicks[b, q]) for q, k in enumerate(("noise", "music"))]
            srcs += [render.Pooled(spk_pool, picks[b, 0], w), render.Pooled(spk_pool, picks[b, 1], w),
                     render.Pooled(noi_pool, picks[b, 2], w, 0, d[0]), render.Pooled(mus_pool, picks[b, 3], w, 0, d[1])]
            mixes.append(render.Mixture([4 * b, 4 * b + 1], [4 * b + 2, 4 * b + 3], sirs[b], snr[b], mix[b], spo[b],
                                        rms[b], mono=True))
        return R.plan_device(srcs, outs, mixtures=mixes)

    plans = {f: plan(f) for f in ("pick", "bed")}

    def step(form):
        picks.copy_(torch.randint(0, SCENES, (B, 4), generator=gen, device=dev, dtype=torch.int32))
        dpicks.copy_(torch.randint(0, 2 * B, (B, 2), generator=gen, device=dev, dtype=torch.int32))
        starts.copy_(torch.randint(0, N - CROP + 1, (B,), generator=gen, device=dev, dtype=torch.int32))
        sirs.uniform_(-6, 6, generator=gen)
        snr.uniform_(10, 20, generator=gen)
        if form == "bed":
            for k in cp:
                for t, v in zip(lay[k], dry.background_audio_layouts(lens[k], N, MM, B, generator=gen)):
                    t.copy_(v)
        plans[form].run()

    times = {f: [] for f in plans}
    for f in plans:                                       # warm-up: graph capture, first launches
        for _ in range(3):
            step(f)
    torch.cuda.synchronize()
    R.check_device_errors()
    for _ in range(ROUNDS):
        for f in plans:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(STEPS):
                step(f)
            e1.record()
            torch.cuda.synchronize()
            times[f].append(e0.elapsed_time(e1) / STEPS)
    R.check_device_errors()
    lt = []
    for _ in range(ROUNDS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(STEPS):
            dry.background_audio_layouts(lens["music"], N, MM, 2 * B, generator=gen)
        e1.record()
        torch.cuda.synchronize()
        lt.append(e0.elapsed_time(e1) / STEPS)
    res = {"device": card(), "B": B, "crop_s": CROP / RATE, "clips": N_CLIP, "m": MM,
           "step_ms": {f: float(np.median(v)) for f, v in times.items()},
           "step_ms_all": times, "layouts_2B_ms": float(np.median(lt))}
    print(json.dumps(res))
    for p in list(plans.values()):
        p.close()


if __name__ == "__main__":
    main()
