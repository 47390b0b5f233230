"""Pair gains in the training step: what it costs to measure the loudness of every (dry signal, candidate) pair once, and
what a dry-picked step costs when every slot stores its stems at its pair's gain.

Workload of time_dry_pool.py (d): a pool of 64 bench.py configs[1] scenes (128 banked moving speakers, P = 40, C = 6,
L = 4096, 30 s, with create_long_audio's 0-10 s gaps before 1-5 s utterances) with mono level tables, 64 banked static
noises, and a dry pool of 256 gappy dry streams of 60 s with level tables; 16 examples per step, each a random scene,
its 2 speakers in random order and its noise, every slot with a dry pick drawn on the device, one 4 s mono crop,
SIRs ~ U(-6, 6), SNRs ~ U(10, 20), one CropDraw per example (tries = 101, threshold -40 dB).
  - Build time (host wall time of Renderer.pair_gains, per pair): the speakers' and the noises' tables over the device
    pools and the device dry pool (256 x 128 and 256 x 64 pairs, SonicSet's U(-19, -15) and U(-26, -22) LUFS), and the
    speakers' table over a host pool and a host dry pool (the first 64 streams: 64 x 128 pairs).
  - Step time: form (d) without pair gains and (p) with them, alternating, 8 rounds x 30 steps, CUDA events around each
    step (median), host wall time per step, and kernels per step (torch.profiler over one step); a check that (p)'s
    stems equal (d)'s times the pairs' (float)gain, bit for bit, with the same drawn starts.
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
N_DRY, DRY_S, N_DRY_HOST = 256, 60, 64
STEPS, ROUNDS = 30, 8


def timed(f):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = f()
    torch.cuda.synchronize()
    return out, 1e3 * (time.perf_counter() - t0)


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(5)
    spk_x = [gaps(rng, x) for x, _, _ in items]
    spk_c = [render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, (_, h, b) in zip(spk_x, items)]
    noi_c = []
    for _ in range(SCENES):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        noi_c.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    streams = [gaps(rng, (rng.standard_normal(DRY_S * RATE) * 0.05).astype(np.float32)) for _ in range(N_DRY)]
    signals = [to(s) for s in streams]
    torch.cuda.synchronize()
    dpool = R.dry_pool(signals, levels=True)
    spk_lv, noi_pool = R.source_pool(spk_c, levels="mono"), R.source_pool(noi_c)
    t_spk = rng.uniform(-19, -15, (N_DRY, len(spk_c)))
    t_noi = rng.uniform(-26, -22, (N_DRY, len(noi_c)))
    pg_spk, ms_spk = timed(lambda: R.pair_gains(spk_lv, dpool, t_spk, sr=RATE))
    pg_noi, ms_noi = timed(lambda: R.pair_gains(noi_pool, dpool, t_noi, sr=RATE))
    # the host form: host banks of the same RIRs, a host pool of the speakers and a host dry pool of the first streams
    host_c = [render.MovingSource(x, R.rir_bank(to(h), host=True), b, b) for x, (_, h, b) in zip(spk_x, items)]
    hpool = R.source_pool(host_c)
    hdry = R.dry_pool(streams[:N_DRY_HOST], host=True)
    pg_host, ms_host = timed(lambda: R.pair_gains(hpool, hdry, t_spk[:N_DRY_HOST], sr=RATE))
    same = np.array_equal(pg_host.loudness, pg_spk.loudness[:N_DRY_HOST])
    pg_host.close()
    hpool.close()
    hdry.close()

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((U, S + 1), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)

    def plan(gains):
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk_lv, picks[e, k], (starts[e], CROP), 0,
                                   render.DryPick(dpool, dpicks[e, k], pg_spk if gains else None)) for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[e], (starts[e], CROP), 0,
                                      render.DryPick(dpool, dpicks[e, S], pg_noi if gains else None)))
        mix, sp, rms = (torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev),
                        torch.empty((U, S), device=dev))
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), outs, starts, u, used

    plan_d, outs_d, starts_d, u_d, used_d = plan(False)
    plan_p, outs_p, starts_p, u_p, used_p = plan(True)

    def choose():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        dpicks.random_(0, N_DRY)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    def step_d():
        choose()
        u_d.uniform_()
        plan_d.run()

    def step_p():
        choose()
        u_p.uniform_()
        plan_p.run()

    forms = (("d", step_d), ("p", step_p))
    for _ in range(3):
        for _, f in forms:
            f()
    # (p)'s stems against (d)'s on the same choices and variates, times the pairs' gains
    choose()
    u_d.uniform_()
    u_p.copy_(u_d)
    plan_d.run()
    plan_p.run()
    torch.cuda.synchronize()
    assert torch.equal(starts_d, starts_p) and torch.equal(used_d, used_p)
    pk, dk, sc = picks.cpu().numpy(), dpicks.cpu().numpy(), scene.cpu().numpy()
    Ls, Ln = pg_spk.loudness, pg_noi.loudness
    for e in range(U):
        for k in range(S + 1):
            g = Ls[dk[e, k], pk[e, k], 1] if k < S else Ln[dk[e, k], sc[e], 1]
            j = (S + 1) * e + k
            assert torch.equal(outs_p[j], outs_d[j] * torch.tensor(np.float32(g), device=dev)), (e, k)
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
    print("workload: pool of %d scenes (bench.py configs[1] with 0-10 s gaps before 1-5 s utterances), dry pool of %d "
          "gappy %d s streams, %d examples per step, %d-sample mono crops, start draws (101 tries); %d rounds x %d steps "
          "per form, alternating" % (SCENES, N_DRY, DRY_S, U, CROP, ROUNDS, STEPS))
    n_s, n_n, n_h = N_DRY * len(spk_c), N_DRY * len(noi_c), N_DRY_HOST * len(spk_c)
    print("build (host wall): speakers %d pairs in %.1f ms (%.4f ms per pair), noises %d pairs in %.1f ms (%.4f ms per "
          "pair), device pools and dry pool; host pool + host dry pool: %d speaker pairs in %.1f ms (%.4f ms per pair), "
          "loudness %s the device form's" % (n_s, ms_spk, ms_spk / n_s, n_n, ms_noi, ms_noi / n_n, n_h, ms_host,
                                             ms_host / n_h, "equal to" if same else "DIFFERENT FROM"))
    print("tables: speakers %d bytes, noises %d bytes" % (pg_spk.nbytes, pg_noi.nbytes))
    names = {"d": "dry picks, no pair gains", "p": "dry picks with pair gains"}
    for (key, _), nl in zip(forms, launches):
        dev_ms, wall_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median; round medians %.4f - %.4f), host wall %.4f ms/step (median "
              "over rounds, %.4f - %.4f), %d kernels per step (profiled step)" %
              (key, names[key], med(dev_ms), min(med(dev_ms[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)),
               max(med(dev_ms[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)), med(wall_ms), min(wall_ms),
               max(wall_ms), nl))
    print("(p) / (d) stream time: %.4f" % (med(res["p"][0]) / med(res["d"][0])))
    print("(p) stems == (d) stems x (float)gain of the picked pairs, bit for bit, same starts and used")
    for p in (plan_d, plan_p, pg_spk, pg_noi, spk_lv, noi_pool, dpool):
        p.close()


if __name__ == "__main__":
    main()
