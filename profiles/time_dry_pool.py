"""Dry picks in the training step: what it costs a pooled step with start draws to take every speaker's dry signal from
a dry pool, picked on the device at every run.

Workload of time_draw_step.py (b): a pool of 64 bench.py configs[1] scenes (128 banked moving speakers, P = 40, C = 6,
L = 4096, 30 s, with create_long_audio's 0-10 s gaps before 1-5 s utterances) with mono level tables, and 64 banked
static noises; 16 examples per step, each a random scene, its 2 speakers in random order and its noise, one 4 s mono
crop, SIRs ~ U(-6, 6), SNRs ~ U(10, 20), one CropDraw per example (tries = 101, threshold -40 dB).  Forms, alternating:
(b) that plan: every speaker renders its candidate's own dry signal, the draw tests the pool's tables;
(d) the same plan where every speaker slot also takes a dry pick (render.DryPick) from a dry pool of 256 gappy dry
    streams of 60 s with level tables: new dry picks are drawn on the device at every step, the draw tests the dry tables.
Per step: stream time (CUDA events around the step, median), host wall time (a run of steps ending in a synchronise,
divided by the steps), kernels per step (torch.profiler over one step).  Also the dry pool's nbytes and build time, and a
check that (d)'s stems equal render_device of the picked candidates with the picked dry signals at the drawn starts, bit
for bit.  Prints the card and its power limit."""
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
from time_draw_step import gaps  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U, SCENES, TRIES, RATE = 4 * 16000, 16, 64, 101, 16000
N_DRY, DRY_S = 256, 60
STEPS, ROUNDS = 30, 8


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
    # 256 dry streams of 60 s: the same gappy layout over white noise at speech-like level
    signals = [to(gaps(rng, (rng.standard_normal(DRY_S * RATE) * 0.05).astype(np.float32))) for _ in range(N_DRY)]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dpool = R.dry_pool(signals, levels=True)
    dry_build_ms = 1e3 * (time.perf_counter() - t0)
    spk_lv, noi_pool = R.source_pool(spk_c, levels="mono"), R.source_pool(noi_c)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)

    def plan(dry):
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk_lv, picks[e, k], (starts[e], CROP), 0,
                                   render.DryPick(dpool, dpicks[e, k]) if dry else None) for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[e], (starts[e], CROP)))
        mix, sp, rms = (torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev),
                        torch.empty((U, S), device=dev))
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), outs, starts, u

    plan_b, _, _, u_b = plan(False)
    plan_d, outs_d, starts_d, u_d = plan(True)

    def choose():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    def step_b():
        choose()
        u_b.uniform_()
        plan_b.run()

    def step_d():
        choose()
        dpicks.random_(0, N_DRY)
        u_d.uniform_()
        plan_d.run()

    forms = (("b", step_b), ("d", step_d))
    for _ in range(3):
        for _, f in forms:
            f()
    # (d)'s stems against render_device of the picked candidates with the picked dry signals at the drawn starts
    step_d()
    torch.cuda.synchronize()
    pk, dk, sc, st = picks.cpu().numpy(), dpicks.cpu().numpy(), scene.cpu().numpy(), starts_d.cpu().numpy()
    srcs = []
    for e in range(U):
        for k in range(S):
            c = spk_c[int(pk[e, k])]
            srcs.append(c._replace(dry=signals[int(dk[e, k])][:N].contiguous(), window=(int(st[e]), CROP)))
        srcs.append(noi_c[int(sc[e])]._replace(window=(int(st[e]), CROP)))
    refs = [torch.empty_like(o) for o in outs_d]
    R.render_device(srcs, refs)
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(outs_d, refs))
    R.check_device_errors()
    launches = []
    for _, f in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        launches.append(sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA))

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: ([], []) for k, _ in forms}
    for _ in range(ROUNDS):
        for key, f in forms:
            dev_ms, wall_ms = res[key]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for e0, e1 in ev:
                e0.record()
                f()
                e1.record()
            torch.cuda.synchronize()
            wall_ms.append(1e3 * (time.perf_counter() - t0) / STEPS)
            dev_ms += [e0.elapsed_time(e1) for e0, e1 in ev]
    R.check_device_errors()
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    print("workload: pool of %d scenes (bench.py configs[1] with 0-10 s gaps before 1-5 s utterances), %d examples per "
          "step, %d-sample mono crops, start draws (101 tries); %d rounds x %d steps per form, alternating"
          % (SCENES, U, CROP, ROUNDS, STEPS))
    print("dry pool: %d streams of %d s with level tables, nbytes %d (%.1f MB), built in %.1f ms (host wall)"
          % (N_DRY, DRY_S, dpool.nbytes, dpool.nbytes / 1e6, dry_build_ms))
    names = {"b": "speakers' own dry signals      ", "d": "every speaker takes a dry pick"}
    for (key, _), nl in zip(forms, launches):
        dev_ms, wall_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median; round medians %.4f - %.4f), host wall %.4f ms/step (median "
              "over rounds, %.4f - %.4f), %d kernels per step (profiled step)" %
              (key, names[key], med(dev_ms), min(med(dev_ms[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)),
               max(med(dev_ms[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)), med(wall_ms), min(wall_ms),
               max(wall_ms), nl))
    print("(d) / (b) stream time: %.4f" % (med(res["d"][0]) / med(res["b"][0])))
    print("(d) stems == render_device of the picked candidates with the picked dry signals, bit for bit")
    for p in (plan_b, plan_d):
        p.close()
    for p in (spk_lv, noi_pool, dpool):
        p.close()


if __name__ == "__main__":
    main()
