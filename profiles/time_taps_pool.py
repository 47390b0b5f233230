"""Tap-form host banks in the training step: what staging RIR taps (Renderer.rir_bank(host=True, form="taps")) and
transforming them on the device costs against staging the spectra of spectral host banks (form="spectra") of the same
RIRs.  Two workloads, each over both forms, alternating in one process:
  (host)  the step of time_host_pool.py: configs[2]-shaped host pools (128 moving speakers, P = 60, C = 6, L = 4096, 30 s,
          over 32 RIR sets; 64 static noises and 64 static musics), 16 examples of 2 pooled speakers + noise + music,
          one drawn 4 s crop and a mono Mixture each;
  (hh)    the step of time_host_dry_pool.py (hh): host pools of 64 configs[1] scenes (P = 40) and 64 static noises,
          every speaker slot dry-picked from a host dry pool of 256 gappy 60 s streams with level tables.
Per step: stream time (CUDA events around the step, median), host wall time, and the library's kernels per step; in
separate runs under torch.profiler, k_stage and the k_prepare launches per step (the tap form's extra k_prepare is the
transform: the difference); bytes staged per run, worked out from the read sets of the drawn picks and starts as
stage_set does (spectra: sets * rows * 32 KB, taps: rows * 16 KB, plus the dry samples); pinned and device bytes of the
pools and banks.  Asserts on the same draws that both forms give identical bits.  Prints the card and its power limit.
Informational: bench.py is unchanged."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from oracle import sonicsim_oracle as so  # noqa: E402
from sonicsim_b200 import render  # noqa: E402
from time_draw_step import gaps  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U, TRIES, RATE, KB = 4 * 16000, 16, 101, 16000, 4096
FORMS = ("spectra", "taps")
STEPS, ROUNDS = 20, 6


def staged_bytes(N, P, C, K, bounds, ws, form, sets):
    """Bytes k_stage copies for one slot of a host pool: stage_set's dry samples as whole float4s and its RIR rows
    [row0, row0 + rows) - sets * 32 KB per row of spectra, 16 KB per row of taps."""
    xa, xb = max(ws - (K + 2) * KB, 0), min(ws + CROP + 2 * KB, N)
    pa = pb = 0
    if P > 1:
        inner = np.asarray(bounds[1:P])
        pa = min(int(np.searchsorted(inner, xa, side="right")), P - 2)
        pb = min(int(np.searchsorted(inner, xb - 1, side="right")), P - 2) + 1
    r0, r1 = (pa * C * K) & ~1, min(((pb + 1) * C * K + 1) & ~1, P * C * K)
    rows = (r1 - r0) * (KB * 4 if form == "taps" else sets * KB * 8)
    return 4 * (((xb + 3) & ~3) - (xa & ~3)) + rows


def to(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def measure(R, name, plans, step, staged, pools):
    """Alternate the forms' steps; print stream / wall time, kernels, profiled k_stage and k_prepare, bytes.  step(f, seed)
    draws the step's picks, starts, SIRs and SNRs from `seed`: both forms run the same seeds, each step a new draw."""
    for i in range(3):                                   # warm-up and graph capture
        for f in FORMS:
            step(f, 1000 + i)
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {f: ([], []) for f in FORMS}
    for r in range(ROUNDS):
        for f in FORMS:
            for i, (e0, e1) in enumerate(ev):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record()
                step(f, 2000 + r * STEPS + i)
                e1.record()
                torch.cuda.synchronize()
                res[f][1].append(1e3 * (time.perf_counter() - t0))
            res[f][0].extend(e0.elapsed_time(e1) for e0, e1 in ev)
    kernels, prof = {}, {}
    for f in FORMS:
        R.reset_stats()
        step(f, 3000)
        torch.cuda.synchronize()
        kernels[f] = R.launch_count()
    for f in FORMS:                                      # each form in a profiler session of its own
        n = 20
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as p:
            for i in range(n):
                step(f, 4000 + i)
            torch.cuda.synchronize()
        tot = {"k_stage": 0.0, "k_prepare": 0.0}
        cnt = {"k_stage": 0, "k_prepare": 0}
        for e in p.events():
            if e.device_type != torch.autograd.DeviceType.CUDA:
                continue
            for k in tot:
                if k in e.name:
                    tot[k] += e.device_time_total
                    cnt[k] += 1
        prof[f] = {k: (tot[k] / n, cnt[k] / n) for k in tot}
    print("[%s]" % name)
    for f in FORMS:
        st, wall = res[f]
        print("  %-7s: stream %.4f ms/step (median of %d; p10 %.4f, p90 %.4f), host wall %.4f ms, %d kernels/step; "
              "k_stage %.1f us, k_prepare %.1f us in %.1f launches per step (torch.profiler); staged %.2f MB per run" %
              (f, np.median(st), len(st), np.percentile(st, 10), np.percentile(st, 90), np.median(wall), kernels[f],
               prof[f]["k_stage"][0], prof[f]["k_prepare"][0], prof[f]["k_prepare"][1], np.median(staged[f]) / 1e6))
    print("  transform (tap form's extra k_prepare time): %.1f us per step" %
          (prof["taps"]["k_prepare"][0] - prof["spectra"]["k_prepare"][0]))
    for f in FORMS:
        for pname, (pl, banks) in pools[f].items():
            print("  %-7s pool %-8s: device %.1f MB, pinned %.1f MB (pool) + %.1f MB (banks)" %
                  (f, pname, pl.nbytes / 1e6, pl.host_nbytes / 1e6, sum(b.host_nbytes for b in banks) / 1e6))


def host_step(R):
    P, C, L, N = 60, 6, 4096, 30 * RATE
    SCENES, RIR_SETS = 64, 32
    rng = np.random.default_rng(2)
    rirs = [so.synth_rirs(rng, P, C, L) for _ in range(RIR_SETS)]
    spk = []
    for j in range(2 * SCENES):
        cuts = np.sort(rng.integers(0, N + 1, P - 2))
        spk.append((so.synth_dry(rng, N), j % RIR_SETS, np.concatenate([[0], cuts, [N]]).astype(np.int32)))
    stat = [(so.synth_dry(rng, N), (rng.standard_normal((C, L)) * np.exp(-np.arange(L) / 800.0)).astype(np.float32))
            for _ in range(2 * SCENES)]
    pools = {}
    for f in FORMS:
        banks = [R.rir_bank(h, host=True, form=f) for h in rirs]
        sb = [R.rir_bank(h, host=True, form=f) for _, h in stat]
        sp = [render.MovingSource(x, banks[r], b, bounds_host=b) for x, r, b in spk]
        st = [render.StaticSource(x, sb[i]) for i, (x, _) in enumerate(stat)]
        pools[f] = {"speakers": (R.source_pool(sp, levels="mono"), banks),
                    "noises": (R.source_pool(st[:SCENES]), sb[:SCENES]),
                    "musics": (R.source_pool(st[SCENES:]), sb[SCENES:])}
    torch.cuda.synchronize()
    picks = torch.zeros((U, 4), dtype=torch.int32, device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
    sirs, snr = torch.zeros((U, 1), device=dev), torch.zeros((U,), device=dev)

    def plan_over(f):
        spk_pool, noi_pool, mus_pool = (pools[f][k][0] for k in ("speakers", "noises", "musics"))
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        stems = torch.empty((U, 4, C, CROP), device=dev)
        mix, out, rms = torch.empty((U, CROP), device=dev), torch.empty((U, 2, CROP), device=dev), \
            torch.empty((U, 2), device=dev)
        srcs, outs, mixes, draws = [], [], [], []
        for e in range(U):
            for k, pl in enumerate((spk_pool, spk_pool, noi_pool, mus_pool)):
                srcs.append(render.Pooled(pl, picks[e, k], (starts[e], CROP)))
                outs.append(stems[e, k])
            mixes.append(render.Mixture([4 * e, 4 * e + 1], [4 * e + 2, 4 * e + 3], sirs[e], snr[e], mix[e], out[e],
                                        rms[e], mono=True))
            draws.append(render.CropDraw(starts[e], [4 * e, 4 * e + 1], u[e]))
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), (stems, mix, out, rms, starts)

    plans = {f: plan_over(f) for f in FORMS}
    gen = torch.Generator(device=dev)

    def step(f, seed):
        gen.manual_seed(seed)
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32, generator=gen)
        picks[:, :2] = 2 * sc[:, None] + torch.rand(U, 2, device=dev, generator=gen).argsort(1).int()
        picks[:, 2] = sc
        picks[:, 3] = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32, generator=gen)
        u.uniform_(generator=gen)
        sirs.uniform_(-6, 6, generator=gen)
        snr.uniform_(10, 20, generator=gen)
        plans[f][0].run()

    staged = {f: [] for f in FORMS}
    for i in range(8):                                   # bits and read sets on the same draws
        for f in FORMS:
            step(f, i)
        torch.cuda.synchronize()
        for a, b in zip(plans["spectra"][1], plans["taps"][1]):
            assert torch.equal(a, b)
        pk, ws = picks.cpu().numpy(), plans["taps"][1][4].cpu().numpy()
        for f in FORMS:
            total = 0
            for e in range(U):
                total += sum(staged_bytes(N, P, C, 1, spk[pk[e, k]][2], int(ws[e]), f, 1) for k in range(2))
                total += 2 * staged_bytes(N, 1, C, 1, None, int(ws[e]), f, 1)
            staged[f].append(total)
    R.check_device_errors()
    measure(R, "host: time_host_pool.py's step", plans, step, staged, pools)
    for f in FORMS:
        plans[f][0].close()
        for pl, banks in pools[f].values():
            pl.close()
            for b in banks:
                b.close()


def hh_step(R):
    SCENES, N_DRY, DRY_S = 64, 256, 60
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    rng = np.random.default_rng(5)
    spk_x = [gaps(rng, x) for x, _, _ in items]
    spk_h = [h for _, h, _ in items]
    spk_b = [b for _, _, b in items]
    P = spk_h[0].shape[0]
    noi_x, noi_h = [], []
    for _ in range(SCENES):
        noi_x.append((rng.standard_normal(N) * 0.05).astype(np.float32))
        noi_h.append((rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32))
    streams = [gaps(rng, (rng.standard_normal(DRY_S * RATE) * 0.05).astype(np.float32)) for _ in range(N_DRY)]
    hpool = R.dry_pool(streams, levels=True, host=True)
    pools = {}
    for f in FORMS:
        sb = [R.rir_bank(h, host=True, form=f) for h in spk_h]
        nb = [R.rir_bank(h, host=True, form=f) for h in noi_h]
        pools[f] = {"speakers": (R.source_pool([render.MovingSource(x, b, bd, bd) for x, b, bd in zip(spk_x, sb, spk_b)]),
                                 sb),
                    "noises": (R.source_pool([render.StaticSource(x, b) for x, b in zip(noi_x, nb)]), nb)}
    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs, snr = torch.zeros((U, S - 1), device=dev), torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)

    def plan(f):
        spk_pool, noi_pool = pools[f]["speakers"][0], pools[f]["noises"][0]
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk_pool, picks[e, k], (starts[e], CROP), 0, render.DryPick(hpool, dpicks[e, k]))
                     for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[e], (starts[e], CROP)))
        mix = torch.empty((U, CROP), device=dev)
        sp, rms = torch.empty((U, S, CROP), device=dev), torch.empty((U, S), device=dev)
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), outs + [starts, used, mix, sp, rms]

    plans = {f: plan(f) for f in FORMS}
    gen = torch.Generator(device=dev)

    def step(f, seed):
        gen.manual_seed(seed)
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32, generator=gen)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev, generator=gen).argsort(1).int())
        scene.copy_(sc)
        sirs.uniform_(-6, 6, generator=gen)
        snr.uniform_(10, 20, generator=gen)
        dpicks.random_(0, N_DRY, generator=gen)
        u.uniform_(generator=gen)
        plans[f][0].run()

    staged = {f: [] for f in FORMS}
    for i in range(8):
        for f in FORMS:
            step(f, i)
        torch.cuda.synchronize()
        for a, b in zip(plans["spectra"][1], plans["taps"][1]):
            assert torch.equal(a, b)
        pk, ws = picks.cpu().numpy(), plans["taps"][1][U * (S + 1)].cpu().numpy()
        for f in FORMS:
            total = 0
            for e in range(U):
                total += sum(staged_bytes(N, P, C, 1, spk_b[pk[e, k]], int(ws[e]), f, 1) for k in range(S))
                total += staged_bytes(N, 1, C, 1, None, int(ws[e]), f, 1)
            staged[f].append(total)
    R.check_device_errors()
    measure(R, "hh: time_host_dry_pool.py's (hh) step", plans, step, staged, pools)
    for f in FORMS:
        plans[f][0].close()
        for pl, banks in pools[f].values():
            pl.close()
            for b in banks:
                b.close()
    hpool.close()


def main():
    R = render.Renderer(0)
    print("device:", card())
    print("workloads: %d examples per step, %d-sample crops, %d-try CropDraws, mono mixtures; %d x %d steps per form, "
          "alternating" % (U, CROP, TRIES, ROUNDS, STEPS))
    host_step(R)
    hh_step(R)
    print("spectral and tap-form host pools give the same bits on the same draws")


if __name__ == "__main__":
    main()
