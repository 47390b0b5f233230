"""Value draws in the training step: what it costs to refresh picks, SIRs, SNRs, crop variates and starts with torch
before every run against drawing them inside the plan (render.ValueDraw, k_values at the head of the run), so that
`rng[1] += 1` is the step's only host-side op.  Both forms draw their layouts in the plan (render.LayoutDraw).

Workloads, both forms of each alternating round by round in one process:
(sd)  time_dry_streams.py's (sd) step: a pool of 64 bench.py configs[1] scenes (128 banked moving speakers, P = 40,
      C = 6, L = 4096, 30 s) and 64 banked static noises; 16 examples per step, each two stream speakers over a 16-bit
      device pool of 2000 utterances of 2 to 20 s (60 s streams, m = 32) and its noise, one 4 s mono crop, SIRs ~
      U(-6, 6), SNRs ~ U(10, 20), one CropDraw per example (101 tries): 32 stream layouts per step.
(bed) time_background_streams.py's (bed) step: 32 of those scenes' speakers and 32 + 32 static noise and music
      candidates; 32 examples per step, each two speakers, a noise bed over a float32 device pool of 300 clips of 10 to
      60 s and a music bed over a 16-bit pinned host pool of 300 clips of 60 s (m = 16): 64 bed layouts per step; plain
      randint crop starts, no CropDraw.
Forms: "torch" refreshes (sd)'s scene, picks (random.sample within the scene), SIRs, SNRs and u, or (bed)'s picks,
starts, SIRs and SNRs with torch ops before plan.run(), as time_layout_draw.py's "plan" form; "values" draws them in
the plan.  Per form: stream time per step (CUDA events around each step, median), kernels per step and k_values' own
time (torch.profiler, separate steps), launches per plan run (ss_launch_count).  Prints the card and its power limit."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from sonicsim_b200 import render  # noqa: E402
from time_host_dry_pool import kernel_ms  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
RATE, CROP = 16000, 4 * 16000
STEPS, ROUNDS = 30, 6


def statics(R, rng, n, C, N, to):
    out = []
    for _ in range(n):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        out.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    return out


def speech(R, to, gen):
    """(sd): {form: step function}, the plans to close."""
    SCENES, U, TRIES, N_UTT, TOTAL, MM = 64, 16, 101, 2000, 60 * RATE, 32
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    rng = np.random.default_rng(5)
    spk = R.source_pool([render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in items])
    noi = R.source_pool(statics(R, rng, SCENES, C, N, to))
    utts = [np.clip(np.round(rng.standard_normal(int(rng.integers(2 * RATE, 20 * RATE))) * 3000 *
                             rng.uniform(0.1, 1.0)), -32768, 32767).astype(np.int16) for _ in range(N_UTT)]
    up = R.dry_pool(utts, levels=True, dtype="int16")
    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs, snr = torch.zeros((U, S - 1), device=dev), torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
    rng_t = torch.tensor([11, 0], dtype=torch.int64, device=dev)
    held = [spk, noi, up]

    def plan(form):
        ids = torch.full((U, S, MM), -1, dtype=torch.int32, device=dev)
        offs = torch.full((U, S, MM), -1, dtype=torch.int32, device=dev)
        starts, used = torch.zeros(U, dtype=torch.int32, device=dev), torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk, picks[e, k], (starts[e], CROP), 0, render.DryStream(up, ids[e, k], offs[e, k]))
                     for k in range(S)]
            srcs.append(render.Pooled(noi, scene[e], (starts[e], CROP)))
        mix = torch.empty((U, CROP), device=dev)
        sp, rms = torch.empty((U, S, CROP), device=dev), torch.empty((U, S), device=dev)
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        layouts = [render.LayoutDraw((S + 1) * e + k, rng_t, TOTAL) for e in range(U) for k in range(S)]
        values = ([render.ValueDraw(scene, rng_t, 0, SCENES),
                   render.ValueDraw(picks, rng_t, 0, S, distinct=True, base=scene, stride=S),
                   render.ValueDraw(sirs, rng_t, -6, 6), render.ValueDraw(snr, rng_t, 10, 20),
                   render.ValueDraw(u, rng_t)] if form == "values" else None)
        p = R.plan_device(srcs, outs, mixtures=mixes, draws=draws, layouts=layouts, values=values)
        held.append(p)
        return p, ids, offs

    def stepper(form):
        p, ids, offs = plan(form)

        def f():
            rng_t[1] += 1
            if form == "torch":
                sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32, generator=gen)
                picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev, generator=gen).argsort(1).int())
                scene.copy_(sc)
                sirs.uniform_(-6, 6, generator=gen)
                snr.uniform_(10, 20, generator=gen)
                u.uniform_(generator=gen)
            p.run()
        return f, p

    return {f: stepper(f) for f in ("torch", "values")}, held


def beds(R, to, gen):
    """(bed): {form: step function}, the plans to close."""
    SCENES, B, N_CLIP, MM = 32, 32, 300, 16
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    rng = np.random.default_rng(7)
    spk = R.source_pool([render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in items])
    noi, mus = R.source_pool(statics(R, rng, SCENES, C, N, to)), R.source_pool(statics(R, rng, SCENES, C, N, to))
    noise = [(rng.standard_normal(int(rng.integers(10 * RATE, 60 * RATE))) * 0.1).astype(np.float32)
             for _ in range(N_CLIP)]
    music = [np.clip(np.round(rng.standard_normal(60 * RATE) * 3000), -32768, 32767).astype(np.int16)
             for _ in range(N_CLIP)]
    cp = {"noise": R.dry_pool([to(c) for c in noise]), "music": R.dry_pool(music, host=True, dtype="int16")}
    picks = torch.zeros((B, 4), dtype=torch.int32, device=dev)
    starts = torch.zeros(B, dtype=torch.int32, device=dev)
    sirs, snr = torch.zeros((B, S - 1), device=dev), torch.zeros(B, device=dev)
    rng_t = torch.tensor([12, 0], dtype=torch.int64, device=dev)
    held = [spk, noi, mus] + list(cp.values())

    def plan(form):
        lay = {k: [torch.full((B, MM), -1, dtype=torch.int32, device=dev) for _ in range(4)] for k in cp}
        outs = [torch.empty((C, CROP), device=dev) for _ in range(4 * B)]
        mix, spo, rms = (torch.empty((B, CROP), device=dev), torch.empty((B, S, CROP), device=dev),
                         torch.empty((B, S), device=dev))
        srcs, mixes, layouts = [], [], []
        for b in range(B):
            w = (starts[b], CROP)
            d = [render.BackgroundStream(cp[k], *[t[b] for t in lay[k]]) for k in ("noise", "music")]
            srcs += [render.Pooled(spk, picks[b, 0], w), render.Pooled(spk, picks[b, 1], w),
                     render.Pooled(noi, picks[b, 2], w, 0, d[0]), render.Pooled(mus, picks[b, 3], w, 0, d[1])]
            mixes.append(render.Mixture([4 * b, 4 * b + 1], [4 * b + 2, 4 * b + 3], sirs[b], snr[b], mix[b], spo[b],
                                        rms[b], mono=True))
            layouts += [render.LayoutDraw(4 * b + 2, rng_t, N), render.LayoutDraw(4 * b + 3, rng_t, N)]
        values = ([render.ValueDraw(picks, rng_t, 0, SCENES), render.ValueDraw(starts, rng_t, 0, N - CROP + 1),
                   render.ValueDraw(sirs, rng_t, -6, 6), render.ValueDraw(snr, rng_t, 10, 20)]
                  if form == "values" else None)
        p = R.plan_device(srcs, outs, mixtures=mixes, layouts=layouts, values=values)
        held.append(p)
        return p, lay

    def stepper(form):
        p, lay = plan(form)

        def f():
            rng_t[1] += 1
            if form == "torch":
                picks.copy_(torch.randint(0, SCENES, (B, 4), generator=gen, device=dev, dtype=torch.int32))
                starts.copy_(torch.randint(0, N - CROP + 1, (B,), generator=gen, device=dev, dtype=torch.int32))
                sirs.uniform_(-6, 6, generator=gen)
                snr.uniform_(10, 20, generator=gen)
            p.run()
        return f, p

    return {f: stepper(f) for f in ("torch", "values")}, held


def measure(R, name, forms):
    for _ in range(3):                                    # warm-up: graph capture, first launches
        for f, _ in forms.values():
            f()
    torch.cuda.synchronize()
    R.check_device_errors()
    out = {}
    for form, (f, p) in forms.items():
        R.reset_stats()
        p.run()
        torch.cuda.synchronize()
        launches = R.launch_count()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                f()
            torch.cuda.synchronize()
        kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA) / 5
        out[form] = {"plan_launches_per_run": launches, "kernels_per_step": kernels,
                     "k_values_ms": kernel_ms(prof, "k_values") / 5,
                     "k_layout_ms": kernel_ms(prof, "k_layout") / 5, "steps_ms": []}
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    for _ in range(ROUNDS):
        for form, (f, _) in forms.items():
            torch.cuda.synchronize()
            for e0, e1 in ev:
                e0.record()
                f()
                e1.record()
            torch.cuda.synchronize()
            out[form]["steps_ms"] += [e0.elapsed_time(e1) for e0, e1 in ev]
    R.check_device_errors()
    for v in out.values():
        v["step_ms_median"] = float(np.median(v.pop("steps_ms")))
    print(json.dumps({"workload": name, "device": card(), **out}))


def main():
    R = render.Renderer(0)
    print("device:", card())
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
    for name, make in (("sd", speech), ("bed", beds)):
        forms, held = make(R, to, gen)
        measure(R, name, forms)
        for h in reversed(held):                          # the plans, then the pools they read
            h.close()
        del forms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
