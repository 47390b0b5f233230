"""Speaker-grouped layout draws in the training step: what it costs to lay each stream out from one speaker's
utterances (render.LayoutDraw(groups=, group=), k_layout_grouped) against from the whole pool (k_layout).

Workload: time_layout_draw.py's (sd) step.  A pool of 64 bench.py configs[1] scenes (128 banked moving speakers,
P = 40, C = 6, L = 4096, 30 s) and 64 banked static noises; 16 examples per step, each two stream speakers over a 16-bit
device pool of 2000 utterances of 2 to 20 s cut into 100 speakers of 10 to 30 utterances (60 s streams, m = 32) and
its noise, one 4 s mono crop, SIRs ~ U(-6, 6), SNRs ~ U(10, 20), one CropDraw per example (101 tries): 32 stream
layouts per step.  Both forms draw each example's two speakers with ValueDraw(spk, rng, 0, 100, distinct=True); only
the grouped form lays its streams out from them.

Both forms alternate round by round in one process.  Per form: stream time per step (CUDA events around each step,
median), kernels per step and the layout kernel's own time (torch.profiler, separate steps), launches per plan run
(ss_launch_count).  Prints the card and its power limit."""
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
    """{form: step function}, the plans and pools to close."""
    SCENES, U, TRIES, TOTAL, MM = 64, 16, 101, 60 * RATE, 32
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    rng = np.random.default_rng(5)
    spk = R.source_pool([render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in items])
    noi = R.source_pool(statics(R, rng, SCENES, C, N, to))
    sizes = rng.integers(10, 31, 100)
    sizes[-1] += 2000 - sizes.sum()                       # 2000 utterances in all
    assert sizes.min() >= 1
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    utts = [np.clip(np.round(rng.standard_normal(int(rng.integers(2 * RATE, 20 * RATE))) * 3000 *
                             rng.uniform(0.1, 1.0)), -32768, 32767).astype(np.int16) for _ in range(int(bounds[-1]))]
    up = R.dry_pool(utts, levels=True, dtype="int16")
    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs, snr = torch.zeros((U, S - 1), device=dev), torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
    rng_t = torch.tensor([11, 0], dtype=torch.int64, device=dev)
    held = [spk, noi, up]

    def plan(form):
        who = torch.zeros((U, S), dtype=torch.int32, device=dev)
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
        g = (lambda e, k: dict(groups=bounds, group=who[e, k:k + 1])) if form == "grouped" else (lambda e, k: {})
        layouts = [render.LayoutDraw((S + 1) * e + k, rng_t, TOTAL, **g(e, k)) for e in range(U) for k in range(S)]
        values = [render.ValueDraw(who, rng_t, 0, len(sizes), distinct=True)]
        p = R.plan_device(srcs, outs, mixtures=mixes, draws=draws, layouts=layouts, values=values)
        held.append(p)
        return p

    def stepper(form):
        p = plan(form)

        def f():
            sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32, generator=gen)
            picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev, generator=gen).argsort(1).int())
            scene.copy_(sc)
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(10, 20, generator=gen)
            u.uniform_(generator=gen)
            rng_t[1] += 1
            p.run()
        return f, p

    return {f: stepper(f) for f in ("ungrouped", "grouped")}, held


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
                     "layout_kernel": "k_layout_grouped" if form == "grouped" else "k_layout",
                     "layout_kernel_ms": kernel_ms(prof, "k_layout") / 5, "steps_ms": []}
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
    forms, held = speech(R, to, gen)
    measure(R, "sd", forms)
    for h in reversed(held):                              # the plans, then the pools they read
        h.close()


if __name__ == "__main__":
    main()
