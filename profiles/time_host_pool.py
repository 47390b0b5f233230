"""What a host pool costs a training step: one step at the configs[2] shape (moving speakers with P = 60 positions, C = 6,
L = 4096, here over 30 s of dry signal) - 64 scenes as pools of 128 banked speakers (2 per scene, over 32 distinct RIR
sets), 64 static noises and 64 static musics (C = 6, L = 4096); 16 examples per step, each 2 pooled speakers + noise +
music, one 4 s crop drawn on the device by a 101-try CropDraw over mono level tables, and a mono Mixture - built once over
device pools and once over host pools of the same candidates (Renderer.rir_bank(host=True): banks, dry signals and level
tables in pinned host memory; k_stage copies each slot's read set to the device at every run).  The two forms alternate
in one process: CUDA events around plan.run(), median over 60 steps each after warm-up.  Also reports k_stage alone
(torch.profiler, its own runs), the bytes it copies per run (worked out here from the read sets of the drawn picks and
starts, as stage_set does) and the rate that gives, the device and host bytes of every pool, the card and its power
limit.  Asserts on the same draws that both forms give the same bits.  Informational: bench.py is unchanged."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
from oracle import sonicsim_oracle as so  # noqa: E402
from sonicsim_b200 import render  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
P, C, L, N, RATE = 60, 6, 4096, 30 * 16000, 16000
SCENES, RIR_SETS, U, CROP, TRIES = 64, 32, 16, 4 * 16000, 101
STEPS, ROUNDS = 10, 6
B = 4096


def read_set_bytes(n, p, k, bounds, ws, length, sets):
    """Bytes k_stage copies for one slot: stage_set's dry samples (whole float4s) and RIR rows of every set."""
    xa, xb = max(0, ws - (k + 2) * B), min(n, ws + length + 2 * B)
    pa = pb = 0
    if p > 1:
        pa = int(np.searchsorted(bounds[1:], xa, side="right"))
        pb = int(np.searchsorted(bounds[1:], xb - 1, side="right")) + 1
    ck = C * k
    r0, r1 = (pa * ck) & ~1, min(((pb + 1) * ck + 1) & ~1, p * ck)
    return 4 * (((xb + 3) & ~3) - (xa & ~3)) + sets * (r1 - r0) * B * 8


def main():
    R = render.Renderer(0)
    print("device:", card())
    rng = np.random.default_rng(2)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rirs = [so.synth_rirs(rng, P, C, L) for _ in range(RIR_SETS)]
    spk = []
    for j in range(2 * SCENES):
        cuts = np.sort(rng.integers(0, N + 1, P - 2))
        spk.append((so.synth_dry(rng, N), j % RIR_SETS, np.concatenate([[0], cuts, [N]]).astype(np.int32)))
    stat = [(so.synth_dry(rng, N), (rng.standard_normal((C, L)) * np.exp(-np.arange(L) / 800.0)).astype(np.float32))
            for _ in range(2 * SCENES)]
    pools = {}
    for host in (False, True):
        banks = [R.rir_bank(h, host=host) for h in rirs]
        sp = [render.MovingSource(x if host else to(x), banks[r], b if host else to(b), bounds_host=b) for x, r, b in spk]
        st = [render.StaticSource(x if host else to(x), R.rir_bank(h, host=host)) for x, h in stat]
        pools[host] = (R.source_pool(sp, levels="mono"), R.source_pool(st[:SCENES]), R.source_pool(st[SCENES:]))
    torch.cuda.synchronize()

    picks = torch.zeros((U, 4), dtype=torch.int32, device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
    sirs, snr = torch.zeros((U, 1), device=dev), torch.zeros((U,), device=dev)

    def plan_over(spk_pool, noi_pool, mus_pool):
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
        plan = R.plan_device(srcs, outs, mixtures=mixes, draws=draws)
        return plan, (stems, mix, out, rms, starts)

    plans = {h: plan_over(*pools[h]) for h in (False, True)}

    def draw():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks[:, :2] = 2 * sc[:, None] + torch.rand(U, 2, device=dev).argsort(1).int()
        picks[:, 2] = sc
        picks[:, 3] = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        u.uniform_()
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    forms = (False, True)
    for _ in range(5):                                   # warm-up and graph capture
        draw()
        for h in forms:
            plans[h][0].run()
    draw()
    for h in forms:
        plans[h][0].run()
    torch.cuda.synchronize()
    for a, b in zip(plans[False][1], plans[True][1]):
        assert torch.equal(a, b)
    R.check_device_errors()

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {h: [] for h in forms}
    staged = []
    for _ in range(ROUNDS):
        for h in forms:
            for e0, e1 in ev:
                draw()
                e0.record()
                plans[h][0].run()
                e1.record()
            torch.cuda.synchronize()
            res[h] += [e0.elapsed_time(e1) for e0, e1 in ev]
            if h:                                    # the bytes of the last step's read sets
                pk, ws = picks.cpu().numpy(), plans[h][1][4].cpu().numpy()
                total = 0
                for e in range(U):
                    for k in range(4):
                        if k < 2:
                            _, r, b = spk[pk[e, k]]
                            total += read_set_bytes(N, P, 1, b, int(ws[e]), CROP, 1)
                        else:
                            total += read_set_bytes(N, 1, 1, None, int(ws[e]), CROP, 1)
                staged.append(total)

    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            draw()
            plans[True][0].run()
        torch.cuda.synchronize()
    ks = [e.device_time_total for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "k_stage" in e.name]
    k_us = float(np.median(ks)) if ks else float("nan")

    med = lambda v: float(np.median(v))                                                     # noqa: E731
    print("workload: %d examples x (2 pooled speakers + noise + music), %d-sample crops, %d-try CropDraw, mono mixtures; "
          "pools over %d scenes (%d speakers P=%d C=%d L=%d N=%d over %d RIR sets, %d noises, %d musics); %d steps per "
          "form, alternating" % (U, CROP, TRIES, SCENES, 2 * SCENES, P, C, L, N, RIR_SETS, SCENES, SCENES,
                                 ROUNDS * STEPS))
    for h in forms:
        print("%s pools: plan.run() %.4f ms/step (median, CUDA events; p10 %.4f, p90 %.4f)" %
              ("host  " if h else "device", med(res[h]), np.percentile(res[h], 10), np.percentile(res[h], 90)))
    mb = med(staged) / 1e6
    print("k_stage alone: %.1f us (median of %d launches, torch.profiler); staged %.2f MB per run (median, from the read "
          "sets) -> %.1f GB/s" % (k_us, len(ks), mb, mb / 1e3 / (k_us * 1e-6) if ks else float("nan")))
    for h in forms:
        for name, pl in zip(("speakers", "noises", "musics"), pools[h]):
            print("%s pool %-8s: device %.1f MB, host %.1f MB" % ("host  " if h else "device", name, pl.nbytes / 1e6,
                                                                   pl.host_nbytes / 1e6))
    print("device and host pools give the same bits on the same draws")
    for h in forms:
        plans[h][0].close()
        for p in pools[h]:
            p.close()


if __name__ == "__main__":
    main()
