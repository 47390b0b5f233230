"""The separation dataloader's training step with its crop start drawn under the silence rule (movingdatamodule.py:81-99).

Workload of time_pool_step.py: a pool of 64 bench.py configs[1] scenes (128 banked moving speakers, P = 40, C = 6,
L = 4096, 30 s) and 64 banked static noises; 16 examples per step, each a random scene, its 2 speakers in random order and
its noise, one 4 s mono crop, SIRs ~ U(-6, 6), SNRs ~ U(10, 20).  The speakers' dry signals get create_long_audio's
layout (SonicSim_audio.py:231-279): 0-10 s of silence before every utterance (here bursts of 1-5 s), so a crop can be
silent.  Forms, alternating:
(a) the pooled plan with uniform starts, ignoring the rule;
(b) a pooled plan with one CropDraw per example (tries = 101, threshold -40 dB): the rule on the device, one graph launch;
(c) today's way of honouring the rule: run (a)'s plan, read rms_db on the host, redraw the starts of the examples with a
    silent speaker and re-run the plan until every example passes (at most 100 redraws, as the dataloader).
Per step: stream time (CUDA events around the step, median), host wall time (a run of steps ending in a synchronise,
divided by the steps), kernels per step (torch.profiler over one step), the share of examples with a speaker below -40 dB
in the plan's rms_db, and for (c) the mean number of re-runs.  Also the level tables' build time per candidate, and a
check that (b)'s stems equal render_device of the picked candidates at the drawn starts, bit for bit.  Prints the card
and its power limit."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from sonicsim_b200 import render  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U, SCENES, TRIES, RATE = 4 * 16000, 16, 64, 101, 16000
STEPS, ROUNDS = 30, 6


def gaps(rng, x):
    """create_long_audio's layout over a dry signal: 0-10 s of silence before every utterance of 1-5 s."""
    y = np.zeros_like(x)
    pos = int(rng.integers(0, 10 * RATE))
    while pos < len(x):
        n = int(rng.integers(RATE, 5 * RATE))
        y[pos:pos + n] = x[pos:pos + n]
        pos += n + int(rng.integers(0, 10 * RATE))
    return y


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(5)
    spk_c = [render.MovingSource(to(gaps(rng, x)), R.rir_bank(to(h)), to(b), b) for x, h, b in items]
    noi_c = []
    for _ in range(SCENES):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        noi_c.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    torch.cuda.synchronize()
    build = []
    for levels in (None, "mono", None, "mono"):
        t0 = time.perf_counter()
        p = R.source_pool(spk_c, levels=levels)
        build.append(time.perf_counter() - t0)
        p.close()
    table_ms = 1e3 * ((build[1] - build[0]) + (build[3] - build[2])) / 2 / len(spk_c)
    spk_pool, spk_lv, noi_pool = R.source_pool(spk_c), R.source_pool(spk_c, levels="mono"), R.source_pool(noi_c)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)

    def plan(pool, starts, u=None, used=None):
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(pool, picks[e, k], (starts[e], CROP)) for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[e], (starts[e], CROP)))
        mix, sp, rms = (torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev),
                        torch.empty((U, S), device=dev))
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = None
        if u is not None:
            draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                     for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), outs, rms

    def choose():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    starts_a = torch.zeros(U, dtype=torch.int32, device=dev)
    plan_a, outs_a, rms_a = plan(spk_pool, starts_a)
    starts_b = torch.zeros(U, dtype=torch.int32, device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
    used = torch.zeros(U, dtype=torch.int32, device=dev)
    plan_b, outs_b, rms_b = plan(spk_lv, starts_b, u, used)
    silent = {"a": [], "b": [], "c": []}
    reruns = []

    def step_a():
        choose()
        starts_a.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        plan_a.run()

    def step_b():
        choose()
        u.uniform_()
        plan_b.run()

    def step_c():
        choose()
        starts_a.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        plan_a.run()
        n = 0
        for _ in range(TRIES - 1):
            bad = rms_a.min(1).values < -40.0
            if not bool(bad.any()):                       # the host reads rms_db: one synchronise per run
                break
            starts_a.copy_(torch.where(bad, torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev),
                                       starts_a))
            plan_a.run()
            n += 1
        reruns.append(n)

    forms = (("a", step_a, rms_a), ("b", step_b, rms_b), ("c", step_c, rms_a))
    for _ in range(3):
        for _, f, _ in forms:
            f()
    # (b)'s stems against render_device of the picked candidates at the drawn starts
    step_b()
    torch.cuda.synchronize()
    pk, sc, st = picks.cpu().numpy(), scene.cpu().numpy(), starts_b.cpu().numpy()
    srcs, refs = [], []
    for e in range(U):
        srcs += [spk_c[int(pk[e, k])]._replace(window=(int(st[e]), CROP)) for k in range(S)]
        srcs.append(noi_c[int(sc[e])]._replace(window=(int(st[e]), CROP)))
    refs = [torch.empty_like(o) for o in outs_b]
    R.render_device(srcs, refs)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs_b, refs))
    R.check_device_errors()
    launches = []
    for _, f, _ in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        launches.append(sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA))
    reruns.clear()

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: ([], []) for k, _, _ in forms}
    for _ in range(ROUNDS):
        for key, f, rms in forms:
            dev_ms, wall_ms = res[key]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            lv = []
            for e0, e1 in ev:
                e0.record()
                f()
                e1.record()
                lv.append(rms.min(1).values.clone())
            torch.cuda.synchronize()
            wall_ms.append(1e3 * (time.perf_counter() - t0) / STEPS)
            dev_ms += [e0.elapsed_time(e1) for e0, e1 in ev]
            silent[key].append(float((torch.stack(lv) < -40.0).float().mean()))
    R.check_device_errors()
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    print("workload: pool of %d scenes (bench.py configs[1] with 0-10 s gaps before 1-5 s utterances), %d examples per "
          "step, %d-sample mono crops, %d rounds x %d steps per form, alternating" % (SCENES, U, CROP, ROUNDS, STEPS))
    print("level tables (mono): %.3f ms per 30 s candidate to build (host wall, pool with tables minus pool without)"
          % table_ms)
    names = {"a": "uniform starts, rule ignored     ", "b": "start draws on the device (101)  ",
             "c": "rms_db to the host, redraw, rerun"}
    for (key, _, _), nl in zip(forms, launches):
        dev_ms, wall_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median), host wall %.4f ms/step (median over rounds, %.4f - %.4f), "
              "%d kernels per step (profiled step), examples with a silent speaker %.2f %%" %
              (key, names[key], med(dev_ms), med(wall_ms), min(wall_ms), max(wall_ms), nl, 100 * np.mean(silent[key])))
    print("(c) mean re-runs per step: %.2f (max %d)" % (np.mean(reruns), max(reruns)))
    print("(b) stems == render_device of the picked candidates at the drawn starts, bit for bit")
    for p in (plan_a, plan_b):
        p.close()
    for p in (spk_pool, spk_lv, noi_pool):
        p.close()


if __name__ == "__main__":
    main()
