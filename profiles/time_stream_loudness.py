"""Loudness slots in the training step: what it costs to store every stream and bed slot at SonicSet's loudness
(render.StemLoudness), measured over its whole stem at every run, against the same step without targets.

Workload: the step of time_background_streams.py with 60 s stems: 64 banked moving speakers (P = 40, C = 6, L = 4096,
60 s) and 32 banked static noise and 32 music candidates (C = 6, 60 s) in device memory; B = 32 examples per step, each
two stream speakers (a 16-bit device pool of 600 utterances of 2 to 20 s, dry.long_audio_layouts, m = 32), a noise
bed (a float32 device pool of 300 clips of 10 to 60 s) and a music bed (a 16-bit pinned host pool of 300 clips of 60 s,
dry.background_audio_layouts, m = 16), one 4 s mono crop per example, SIRs ~ U(-6, 6), SNRs ~ U(10, 20).  Forms,
alternating round by round in one process:
(plain) the step without targets;
(lufs)  every slot with a StemLoudness, targets refreshed before every step: speakers U(-19, -15), noise U(-26, -22),
        music U(-31, -27).
Per step: stream time (CUDA events around the step, median over rounds), layouts and targets refreshed inside it.  Then
kernel times per step from a separate torch.profiler run of each form, and the plan scratch the loudness slots add.
Prints the card and its power limit, and one JSON line, also written to the file named by the first argument if given."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from sonicsim_b200 import dry, render  # noqa: E402
from sonicsim_b200.SonicSim_audio import gating_plan  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
RATE = 16000
N, CROP, B, SCENES, C, P = 60 * RATE, 4 * RATE, 32, 32, 6, 40
N_UTT, N_CLIP, MS, MB = 600, 300, 32, 16
STEPS, ROUNDS, PROF_STEPS = 5, 6, 3


def main():
    R = render.Renderer(0)
    print("device:", card())
    rng = np.random.default_rng(7)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    decay = np.exp(-np.arange(4096) / 800.0)

    def rirs(p):
        return (rng.standard_normal((p, C, 4096)) * decay).astype(np.float32)

    bounds = np.round(np.linspace(0, N, P)).astype(np.int32)
    spk_pool = R.source_pool([render.MovingSource(to((rng.standard_normal(N) * 0.05).astype(np.float32)),
                                                  R.rir_bank(to(rirs(P))), to(bounds), bounds)
                              for _ in range(2 * SCENES)])
    noi_pool, mus_pool = [R.source_pool([render.StaticSource(to((rng.standard_normal(N) * 0.05).astype(np.float32)),
                                                             R.rir_bank(to(rirs(1)[0]))) for _ in range(SCENES)])
                          for _ in range(2)]
    utts = [np.clip(np.round(rng.standard_normal(int(rng.integers(2 * RATE, 20 * RATE))) * 3000), -32768,
                    32767).astype(np.int16) for _ in range(N_UTT)]
    noise = [(rng.standard_normal(int(rng.integers(10 * RATE, 60 * RATE))) * 0.1).astype(np.float32)
             for _ in range(N_CLIP)]
    music = [np.clip(np.round(rng.standard_normal(60 * RATE) * 3000), -32768, 32767).astype(np.int16)
             for _ in range(N_CLIP)]
    up = R.dry_pool(utts, dtype="int16")
    cp = {"noise": R.dry_pool([to(c) for c in noise]), "music": R.dry_pool(music, host=True, dtype="int16")}
    ulen = torch.tensor([u.size for u in utts], device=dev)
    lens = {"noise": torch.tensor([c.size for c in noise], device=dev),
            "music": torch.tensor([c.size for c in music], device=dev)}
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
    sids = torch.full((B, 2, MS), -1, dtype=torch.int32, device=dev)
    soffs = torch.zeros((B, 2, MS), dtype=torch.int32, device=dev)
    lay = {k: [torch.full((B, MB), -1, dtype=torch.int32, device=dev) for _ in range(4)] for k in cp}
    picks = torch.zeros((B, 4), dtype=torch.int32, device=dev)
    starts = torch.zeros(B, dtype=torch.int32, device=dev)
    sirs, snr = torch.zeros((B, 1), device=dev), torch.zeros(B, device=dev)
    lufs = torch.zeros((B, 4), dtype=torch.float64, device=dev)
    outs = [torch.empty((C, CROP), device=dev) for _ in range(4 * B)]
    mix, spo, rms = (torch.empty((B, CROP), device=dev), torch.empty((B, 2, CROP), device=dev),
                     torch.empty((B, 2), device=dev))

    def plan(form):
        srcs, mixes = [], []
        for b in range(B):
            w = (starts[b], CROP)
            q = [render.StemLoudness(lufs[b, k:k + 1]) if form == "lufs" else None for k in range(4)]
            srcs += [render.Pooled(spk_pool, picks[b, k], w, 0, render.DryStream(up, sids[b, k], soffs[b, k], q[k]))
                     for k in range(2)]
            srcs += [render.Pooled(pl, picks[b, 2 + j], w, 0,
                                   render.BackgroundStream(cp[k], *[t[b] for t in lay[k]], lufs=q[2 + j]))
                     for j, (pl, k) in enumerate(((noi_pool, "noise"), (mus_pool, "music")))]
            mixes.append(render.Mixture([4 * b, 4 * b + 1], [4 * b + 2, 4 * b + 3], sirs[b], snr[b], mix[b], spo[b],
                                        rms[b], mono=True))
        return R.plan_device(srcs, outs, mixtures=mixes)

    plans = {f: plan(f) for f in ("plain", "lufs")}

    def step(form):
        picks.copy_(torch.randint(0, SCENES, (B, 4), generator=gen, device=dev, dtype=torch.int32))
        starts.copy_(torch.randint(0, N - CROP + 1, (B,), generator=gen, device=dev, dtype=torch.int32))
        sirs.uniform_(-6, 6, generator=gen)
        snr.uniform_(10, 20, generator=gen)
        a, o = dry.long_audio_layouts(ulen, N, MS, 2 * B, generator=gen)
        sids.copy_(a.view(B, 2, MS))
        soffs.copy_(o.view(B, 2, MS))
        for k in cp:
            for t, v in zip(lay[k], dry.background_audio_layouts(lens[k], N, MB, B, generator=gen)):
                t.copy_(v.view(B, MB))
        if form == "lufs":
            lufs[:, :2].uniform_(-19, -15, generator=gen)
            lufs[:, 2].uniform_(-26, -22, generator=gen)
            lufs[:, 3].uniform_(-31, -27, generator=gen)
        plans[form].run()

    R.reset_stats()
    launches = {}
    for f in plans:                                       # warm-up: graph capture, first launches
        for _ in range(3):
            step(f)
        torch.cuda.synchronize()
        before = R.launch_count()
        plans[f].run()
        torch.cuda.synchronize()
        launches[f] = R.launch_count() - before
    R.check_device_errors()
    times = {f: [] for f in plans}
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

    kernels = {}
    for f in plans:                                       # kernel times: a profiled run of its own per form
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(PROF_STEPS):
                step(f)
            torch.cuda.synchronize()
        agg = {}
        for e in prof.events():
            if e.device_type == torch.autograd.DeviceType.CUDA:
                name = e.name.split("(")[0].replace("void ", "")
                agg[name] = agg.get(name, 0.0) + e.device_time_total / 1000.0 / PROF_STEPS
        kernels[f] = {k: round(v, 4) for k, v in sorted(agg.items(), key=lambda kv: -kv[1]) if v > 0.001}

    brk = gating_plan(N, float(RATE), 0.4)[0]
    n_e = len(brk) - 1
    up256 = lambda v: (v + 255) // 256 * 256                                                # noqa: E731
    per_slot = up256(4 * C * N) + up256(8 * 20 * C * n_e) + 256       # whole stem, loudness scratch, result
    res = {"device": card(), "B": B, "stem_s": N / RATE, "crop_s": CROP / RATE, "C": C,
           "step_ms": {f: float(np.median(v)) for f, v in times.items()}, "step_ms_all": times,
           "launches_per_run": launches, "kernel_ms_per_step": kernels,
           "loudness_slots": 4 * B, "scratch_bytes_per_slot": per_slot, "scratch_bytes": 4 * B * per_slot}
    line = json.dumps(res)
    print(line)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as fh:
            fh.write(line + "\n")
    for p in plans.values():
        p.close()


if __name__ == "__main__":
    main()
