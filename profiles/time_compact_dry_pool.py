"""16-bit dry pools in the training step: what it costs to hold the dry pool of the step of time_dry_pool.py (d) as int16
samples with sparse level tables (Renderer.dry_pool(..., dtype="int16")) instead of float32 with full tables.

Workload of time_dry_pool.py (d) (DESIGN section 6): a pool of 64 bench.py configs[1] scenes (128 banked moving speakers,
P = 40, C = 6, L = 4096, 30 s) and 64 banked static noises in device memory; 16 examples per step, each a random scene,
its 2 speakers in random order and its noise, one 4 s mono crop, SIRs ~ U(-6, 6), SNRs ~ U(10, 20), one CropDraw per
example (tries = 101, threshold -40 dB) over the dry tables; every speaker slot (32 per step) takes a dry pick from 256
gappy 60 s dry streams on the int16 grid, with level tables.  Forms, alternating round by round:
(fd) float32 dry pool in device memory;    (id) 16-bit dry pool in device memory (k_stage<true> stages the crops);
(fh) float32 dry pool in pinned host memory; (ih) 16-bit dry pool in pinned host memory.
Per step: stream time (CUDA events around the step, median) and host wall time; kernels per step and the k_stage and
k_draw times (torch.profiler, separate steps); bytes k_stage reads per run (from the read sets of the drawn starts).
Checks that every form's stems, starts, `used` and mixtures equal (fd)'s bit for bit.  Then builds 1024 x 60 s pools of
each form (one stream given 1024 times: every pool copies or references each) and reports build time and device and
pinned bytes.  Prints the card and its power limit."""
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
from time_host_dry_pool import kernel_ms  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U, SCENES, TRIES, RATE = 4 * 16000, 16, 64, 101, 16000
N_DRY, DRY_S, N_BIG = 256, 60, 1024
STEPS, ROUNDS = 30, 8
KB = 4096
FORMS = ("fd", "id", "fh", "ih")


def read_span(N, K, ws):
    """Dry samples k_stage reads for one dry-picked slot: whole groups of 4 around stage_set's [xa, xb)."""
    xa, xb = max(ws - (K + 2) * KB, 0), min(ws + CROP + 2 * KB, N)
    return ((xb + 3) & ~3) - (xa & ~3)


def to_grid(x):
    """int16 samples of x (the stream as 16-bit PCM)."""
    return np.clip(np.round(x.astype(np.float64) * 32768), -32768, 32767).astype(np.int16)


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(5)
    spk_c = [render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in items]
    noi_c = []
    for _ in range(SCENES):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        noi_c.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    k16 = [to_grid(gaps(rng, (rng.standard_normal(DRY_S * RATE) * 0.1).astype(np.float32))) for _ in range(N_DRY)]
    fl = [k.astype(np.float32) / np.float32(32768) for k in k16]
    torch.cuda.synchronize()
    dry = {"fd": R.dry_pool([to(x) for x in fl], levels=True), "id": R.dry_pool(k16, levels=True, dtype="int16"),
           "fh": R.dry_pool(fl, levels=True, host=True), "ih": R.dry_pool(k16, levels=True, host=True, dtype="int16")}
    spk, noi = R.source_pool(spk_c), R.source_pool(noi_c)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)

    def plan(dp):
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk, picks[e, k], (starts[e], CROP), 0, render.DryPick(dp, dpicks[e, k]))
                     for k in range(S)]
            srcs.append(render.Pooled(noi, scene[e], (starts[e], CROP)))
        mix = torch.empty((U, CROP), device=dev)
        sp, rms = torch.empty((U, S, CROP), device=dev), torch.empty((U, S), device=dev)
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), dict(outs=outs, starts=starts, used=used,
                                                                             mix=mix, sp=sp, rms=rms)

    plans = {k: plan(dry[k]) for k in FORMS}

    def choose():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)
        dpicks.random_(0, N_DRY)
        u.uniform_()

    def stepper(key):
        def f():
            choose()
            plans[key][0].run()
        return f

    forms = [(k, stepper(k)) for k in FORMS]
    for _ in range(3):
        for _, f in forms:
            f()
    # the four forms on the same inputs: equal stems, starts, used and mixtures
    n_checked = 0
    for _ in range(4):
        choose()
        for k in FORMS:
            plans[k][0].run()
        torch.cuda.synchronize()
        for k in FORMS[1:]:
            a, b = plans[k][1], plans["fd"][1]
            for name in ("starts", "used", "mix", "sp", "rms"):
                assert torch.equal(a[name], b[name]), (k, name)
            assert all(torch.equal(x, y) for x, y in zip(a["outs"], b["outs"])), k
            n_checked += 1
    R.check_device_errors()
    st = plans["fd"][1]["starts"].cpu().numpy()
    samples = sum(read_span(N, 1, int(st[e])) for e in range(U) for _ in range(S))
    launches, stage_ms, draw_ms = {}, {}, {}
    for key, f in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                f()
            torch.cuda.synchronize()
        launches[key] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA) / 5
        stage_ms[key] = kernel_ms(prof, "k_stage") / 5
        draw_ms[key] = kernel_ms(prof, "k_draw") / 5

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
    print("workload: time_dry_pool.py (d): pool of %d scenes, %d examples per step (%d dry-picked speaker crops of %d "
          "samples), start draws (101 tries) over the dry tables, dry picks from %d streams of %d s on the int16 grid; "
          "%d rounds x %d steps per form, alternating" % (SCENES, U, U * S, CROP, N_DRY, DRY_S, ROUNDS, STEPS))
    for k in FORMS:
        print("dry pool (%s): nbytes %d (%.1f MB), host_nbytes %d (%.1f MB), level_stride %d" %
              (k, dry[k].nbytes, dry[k].nbytes / 1e6, dry[k].host_nbytes, dry[k].host_nbytes / 1e6,
               dry[k].level_stride))
    names = {"fd": "float32, device", "id": "16-bit, device ", "fh": "float32, host  ", "ih": "16-bit, host   "}
    for key, _ in forms:
        dev_ms, wall_ms = res[key]
        rm = [med(dev_ms[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)]
        staged = "nothing" if key == "fd" else "%.2f MB/run read (%d dry samples x %d B)" % (
            samples * (2 if key[0] == "i" else 4) / 1e6, samples, 2 if key[0] == "i" else 4)
        print("(%s) %s: stream time %.4f ms/step (median; round medians %.4f - %.4f), host wall %.4f ms/step, "
              "%d kernels per step, k_stage %.4f ms/step, k_draw %.4f ms/step (profiled), k_stage %s" %
              (key, names[key], med(dev_ms), min(rm), max(rm), med(wall_ms), launches[key], stage_ms[key],
               draw_ms[key], staged))
    for key in FORMS[1:]:
        print("(%s) - (fd) stream time: %+.4f ms/step, (%s) / (fd): %.4f" %
              (key, med(res[key][0]) - med(res["fd"][0]), key, med(res[key][0]) / med(res["fd"][0])))
    print("(id), (fh) and (ih) stems, starts, used, speakers_out, rms_db and mixtures == (fd), bit for bit (%d checks)"
          % n_checked)
    for p, _ in plans.values():
        p.close()
    for p in list(dry.values()) + [spk, noi]:
        p.close()

    # 1024 x 60 s pools with tables
    avail = 0
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    one_f, one_k = fl[0], k16[0]
    for key in ("id", "ih", "fd", "fh"):
        pinned = {"ih": 2.125, "fh": 12.0}.get(key, 0.0) * N_BIG * DRY_S * RATE
        if pinned and avail < 2 * pinned:
            print("1024 x 60 s pool (%s): not measured (MemAvailable %.1f GB)" % (key, avail / 1e9))
            continue
        given = ([to(one_f)] * N_BIG if key == "fd" else [one_f] * N_BIG if key == "fh" else [one_k] * N_BIG)
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        t0 = time.perf_counter()
        big = R.dry_pool(given, levels=True, host=key[1] == "h", dtype="int16" if key[0] == "i" else "float32")
        build_s = time.perf_counter() - t0
        free1 = torch.cuda.mem_get_info()[0]
        print("1024 x 60 s pool (%s): nbytes %.3f GB, host_nbytes %.3f GB, built in %.2f s (host wall), device free "
              "memory %+.1f MB%s" % (key, big.nbytes / 1e9, big.host_nbytes / 1e9, build_s, (free1 - free0) / 2 ** 20,
                                    " (the 1024 signals reference one tensor)" if key == "fd" else ""))
        big.close()
        del given


if __name__ == "__main__":
    main()
