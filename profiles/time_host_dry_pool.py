"""Host dry pools in the training step: what it costs to keep the dry pool of the step of time_dry_pool.py (d) in pinned
host memory, staged by k_stage at every run, instead of in device memory.

Workload of time_dry_pool.py (d): a pool of 64 bench.py configs[1] scenes (128 banked moving speakers, P = 40, C = 6,
L = 4096, 30 s, with 0-10 s gaps before 1-5 s utterances) and 64 banked static noises; 16 examples per step, each a
random scene, its 2 speakers in random order and its noise, one 4 s mono crop, SIRs ~ U(-6, 6), SNRs ~ U(10, 20), one
CropDraw per example (tries = 101, threshold -40 dB) over the dry tables; every speaker slot takes a dry pick from 256
gappy dry streams of 60 s with level tables.  Forms, alternating:
(d)  the dry pool in device memory;
(h)  the same dry pool with host=True: k_stage copies each speaker slot's dry read set at every run;
(hh) host source pools (host banks) for speakers and noises, plus the host dry pool.
Per step: stream time (CUDA events around the step, median), host wall time, kernels per step and k_stage's time
(torch.profiler over separate steps), bytes staged per run (from the read sets of the drawn starts and picks), and the
device and pinned bytes of each pool.  Also checks that (h)'s and (hh)'s stems, starts and mixtures equal (d)'s bit for
bit, and times the build of a larger host dry pool (1024 streams of 60 s with tables) when the host has the memory.
Prints the card and its power limit."""
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
N_DRY, DRY_S, N_BIG = 256, 60, 1024
STEPS, ROUNDS = 30, 8
KB = 4096


def stage_bytes(N, P, C, K, bounds, ws, rows):
    """Bytes k_stage copies for one slot (stage_set of ss_phases.cuh): the dry samples as whole float4s, and with `rows`
    the RIR rows of the positions they reach (32 KB per half-spectrum row)."""
    xa, xb = max(ws - (K + 2) * KB, 0), min(ws + CROP + 2 * KB, N)
    b = 4 * (((xb + 3) & ~3) - (xa & ~3))
    if rows:
        pa = pb = 0
        if P > 1:
            inner = np.asarray(bounds[1:P])
            pa = min(int(np.searchsorted(inner, xa, side="right")), P - 2)
            pb = min(int(np.searchsorted(inner, xb - 1, side="right")), P - 2) + 1
        r0, r1 = (pa * C * K) & ~1, min(((pb + 1) * C * K + 1) & ~1, P * C * K)
        b += (r1 - r0) * KB * 8
    return b


def kernel_ms(prof, name):
    tot = 0.0
    for e in prof.key_averages():
        if name in e.key:
            tot += getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0.0))
    return tot / 1e3


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(5)
    spk_x = [gaps(rng, x) for x, _, _ in items]
    spk_h = [h for _, h, _ in items]
    spk_b = [b for _, _, b in items]
    noi_x, noi_h = [], []
    for _ in range(SCENES):
        noi_x.append((rng.standard_normal(N) * 0.05).astype(np.float32))
        noi_h.append((rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32))
    spk_c = [render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in zip(spk_x, spk_h, spk_b)]
    noi_c = [render.StaticSource(to(x), R.rir_bank(to(h))) for x, h in zip(noi_x, noi_h)]
    spk_hc = [render.MovingSource(x, R.rir_bank(h, host=True), b, b) for x, h, b in zip(spk_x, spk_h, spk_b)]
    noi_hc = [render.StaticSource(x, R.rir_bank(h, host=True)) for x, h in zip(noi_x, noi_h)]
    streams = [gaps(rng, (rng.standard_normal(DRY_S * RATE) * 0.05).astype(np.float32)) for _ in range(N_DRY)]
    signals = [to(x) for x in streams]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    dpool = R.dry_pool(signals, levels=True)
    d_build = 1e3 * (time.perf_counter() - t0)
    t0 = time.perf_counter()
    hpool = R.dry_pool(streams, levels=True, host=True)
    h_build = 1e3 * (time.perf_counter() - t0)
    spk_dev, noi_dev = R.source_pool(spk_c, levels="mono"), R.source_pool(noi_c)
    spk_host, noi_host = R.source_pool(spk_hc), R.source_pool(noi_hc)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)

    def plan(spk_pool, noi_pool, dry):
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk_pool, picks[e, k], (starts[e], CROP), 0, render.DryPick(dry, dpicks[e, k]))
                     for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[e], (starts[e], CROP)))
        mix = torch.empty((U, CROP), device=dev)
        sp, rms = torch.empty((U, S, CROP), device=dev), torch.empty((U, S), device=dev)
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), dict(outs=outs, starts=starts, used=used,
                                                                             mix=mix)

    plans = {"d": plan(spk_dev, noi_dev, dpool), "h": plan(spk_dev, noi_dev, hpool),
             "hh": plan(spk_host, noi_host, hpool)}

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

    forms = [(k, stepper(k)) for k in ("d", "h", "hh")]
    for _ in range(3):
        for _, f in forms:
            f()
    # the three forms on the same inputs: equal stems, starts and mixtures
    choose()
    for k in ("d", "h", "hh"):
        plans[k][0].run()
    torch.cuda.synchronize()
    for k in ("h", "hh"):
        a, b = plans[k][1], plans["d"][1]
        assert torch.equal(a["starts"], b["starts"]) and torch.equal(a["used"], b["used"]) and \
            torch.equal(a["mix"], b["mix"]) and all(torch.equal(x, y) for x, y in zip(a["outs"], b["outs"])), k
    R.check_device_errors()
    # bytes staged per run, from the read sets of these starts and picks
    pk, sc, st = picks.cpu().numpy(), scene.cpu().numpy(), plans["d"][1]["starts"].cpu().numpy()
    staged = {"h": 0, "hh": 0}
    for e in range(U):
        for k in range(S):
            i = int(pk[e, k])
            staged["h"] += stage_bytes(N, 40, C, 1, spk_b[i], int(st[e]), False)
            staged["hh"] += stage_bytes(N, 40, C, 1, spk_b[i], int(st[e]), True)
        staged["hh"] += stage_bytes(N, 1, C, 1, None, int(st[e]), True)
    launches, stage_ms = {}, {}
    for key, f in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                f()
            torch.cuda.synchronize()
        launches[key] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA) / 5
        stage_ms[key] = kernel_ms(prof, "k_stage") / 5

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
    print("workload: time_dry_pool.py (d): pool of %d scenes, %d examples per step, %d-sample mono crops, start draws "
          "(101 tries) over the dry tables, every speaker dry-picked from %d streams of %d s; %d rounds x %d steps per "
          "form, alternating" % (SCENES, U, CROP, N_DRY, DRY_S, ROUNDS, STEPS))
    print("dry pool, device: nbytes %d (%.1f MB), built in %.1f ms (host wall)" % (dpool.nbytes, dpool.nbytes / 1e6,
                                                                                  d_build))
    print("dry pool, host:   nbytes %d, host_nbytes %d (%.1f MB pinned), built in %.1f ms (host wall, copies included)"
          % (hpool.nbytes, hpool.host_nbytes, hpool.host_nbytes / 1e6, h_build))
    for name, p in (("speaker pool, device", spk_dev), ("noise pool, device", noi_dev), ("speaker pool, host", spk_host),
                    ("noise pool, host", noi_host)):
        print("%s: nbytes %d (%.1f MB), host_nbytes %d (%.1f MB)" % (name, p.nbytes, p.nbytes / 1e6, p.host_nbytes,
                                                                     p.host_nbytes / 1e6))
    names = {"d": "device dry pool               ", "h": "host dry pool                 ",
             "hh": "host source pools + host dry  "}
    for key, _ in forms:
        dev_ms, wall_ms = res[key]
        rm = [med(dev_ms[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)]
        print("(%s) %s: stream time %.4f ms/step (median; round medians %.4f - %.4f), host wall %.4f ms/step, "
              "%d kernels per step, k_stage %.4f ms/step (profiled), staged %s" %
              (key, names[key], med(dev_ms), min(rm), max(rm), med(wall_ms), launches[key], stage_ms[key],
               "%.2f MB/run (%.3f MB per speaker slot)" % (staged[key] / 1e6, staged["h"] / 1e6 / (U * S))
               if key in staged else "nothing"))
    for key in ("h", "hh"):
        print("(%s) - (d) stream time: %+.4f ms/step, (%s) / (d): %.4f" % (key, med(res[key][0]) - med(res["d"][0]),
                                                                          key, med(res[key][0]) / med(res["d"][0])))
    print("(h) and (hh) stems, starts and mixtures == (d), bit for bit")
    for p, _ in plans.values():
        p.close()
    for p in (spk_dev, noi_dev, spk_host, noi_host, dpool, hpool):
        p.close()

    # a larger host dry pool: 1024 streams of 60 s with tables (one stream given 1024 times: the pool copies each)
    need = N_BIG * DRY_S * RATE * 12
    avail = 0
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    if avail < 2 * need:
        print("large host dry pool: not measured (MemAvailable %.1f GB, needs %.1f GB pinned)" % (avail / 1e9, need / 1e9))
        return
    free0 = torch.cuda.mem_get_info()[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    big = R.dry_pool([streams[0]] * N_BIG, levels=True, host=True)
    build_s = time.perf_counter() - t0
    free1 = torch.cuda.mem_get_info()[0]
    print("large host dry pool: %d streams of %d s with tables, host_nbytes %.2f GB (signal %.2f GB, tables %.2f GB), "
          "nbytes %d, built in %.2f s (host wall), device free memory %+.1f MB; MemAvailable before %.1f GB" %
          (N_BIG, DRY_S, big.host_nbytes / 1e9, N_BIG * DRY_S * RATE * 4 / 1e9, N_BIG * (DRY_S * RATE + 1) * 8 / 1e9,
           big.nbytes, build_s, (free1 - free0) / 2 ** 20, avail / 1e9))
    big.close()


if __name__ == "__main__":
    main()
