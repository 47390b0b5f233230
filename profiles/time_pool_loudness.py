"""What loudness gains cost a pooled training step: the workload of time_pool_step.py (b) - 64 bench.py configs[1] scenes
as a pool of 128 banked moving speakers (P = 40, C = 6, L = 4096, 30 s) and 64 banked static noises, 16 examples per
step, each a random scene, its 2 speakers in random order and its noise, one 4 s crop with a new start, SIRs, SNRs and
mono mixtures, all drawn on the device, one graph launch per step - over pools with gains (Renderer.source_pool(...,
lufs_targets=): speakers ~ U(-19, -15) LUFS, noises ~ U(-26, -22), as SonicSet stores them) against the same pools without
them.  The two forms alternate.  Per step: stream time (CUDA events, median), host wall time (a run of steps back to back
ending in a synchronise, divided by the steps) and kernel launches (torch.profiler over one step).  Build cost: the wall
time of source_pool with targets minus without, per 30 s candidate (ss_pool_loudness renders and measures every
candidate once), median of 3 builds.  Asserts in the same run that on the same draws every gained stem is the ungained
stem times its candidate's float32 gain, bit for bit.  Prints the card and its power limit.  Informational: bench.py is
unchanged."""
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
CROP, U, SCENES = 4 * 16000, 16, 64
STEPS, ROUNDS = 50, 8


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
    t_spk = list(rng.uniform(-19, -15, len(spk_c)))
    t_noi = list(rng.uniform(-26, -22, len(noi_c)))

    def build(targets):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        sp = R.source_pool(spk_c, lufs_targets=targets[0] if targets else None)
        npl = R.source_pool(noi_c, lufs_targets=targets[1] if targets else None)
        torch.cuda.synchronize()
        return sp, npl, time.perf_counter() - t0

    costs = []
    for _ in range(3):
        for targets in ((t_spk, t_noi), None):
            sp, npl, t = build(targets)
            costs.append((targets is not None, t))
            sp.close()
            npl.close()
    with_t = float(np.median([t for g, t in costs if g]))
    without_t = float(np.median([t for g, t in costs if not g]))
    per_cand_ms = 1e3 * (with_t - without_t) / (len(spk_c) + len(noi_c))

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    starts = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)

    def plan_over(spk_pool, noi_pool):
        spk = torch.empty((U, S, C, CROP), device=dev)
        noi = torch.empty((U, 1, C, CROP), device=dev)
        outs, srcs = [], []
        for u in range(U):
            outs += [spk[u, k] for k in range(S)] + [noi[u, 0]]
            srcs += [render.Pooled(spk_pool, picks[u, k], (starts[u], CROP)) for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[u], (starts[u], CROP)))
        mix, out, rms = torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev), \
            torch.empty((U, S), device=dev)
        mixes = [render.Mixture(list(range((S + 1) * u, (S + 1) * u + S)), [(S + 1) * u + S], sirs[u], snr[u], mix[u],
                                out[u], rms[u], mono=True) for u in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes), spk, noi

    pools = {"g": build((t_spk, t_noi))[:2], "p": build(None)[:2]}
    plans = {k: plan_over(*v) for k, v in pools.items()}

    def draw():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        starts.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    def step(key):
        draw()
        plans[key][0].run()

    def check_same_draws():
        """The gained plan's stems are the ungained plan's times each picked candidate's float32 gain, bit for bit."""
        draw()
        plans["g"][0].run()
        plans["p"][0].run()
        torch.cuda.synchronize()
        gs = torch.from_numpy(pools["g"][0].loudness[:, 1].astype(np.float32)).to(dev)
        gn = torch.from_numpy(pools["g"][1].loudness[:, 1].astype(np.float32)).to(dev)
        want_s = plans["p"][1] * gs[picks.long()][:, :, None, None]
        want_n = plans["p"][2] * gn[scene.long()][:, None, None, None]
        assert torch.equal(plans["g"][1], want_s) and torch.equal(plans["g"][2], want_n)

    forms = ("g", "p")
    for _ in range(5):                                   # warm-up and graph capture
        for k in forms:
            step(k)
    check_same_draws()
    R.check_device_errors()
    launches = {}
    for k in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            step(k)
            torch.cuda.synchronize()
        launches[k] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: ([], []) for k in forms}
    for _ in range(ROUNDS):
        for k in forms:
            dev_ms, wall_ms = res[k]
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for e0, e1 in ev:
                e0.record()
                step(k)
                e1.record()
            torch.cuda.synchronize()
            wall_ms.append(1e3 * (time.perf_counter() - t0) / STEPS)
            dev_ms += [e0.elapsed_time(e1) for e0, e1 in ev]
    check_same_draws()
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    print("workload: time_pool_step.py (b): pool of %d scenes (%d banked speakers, %d banked static noises, 30 s), %d "
          "examples per step, %d-sample mono crops, mixtures; %d rounds x %d steps per form, alternating" %
          (SCENES, S * SCENES, SCENES, U, CROP, ROUNDS, STEPS))
    names = {"g": "pools with gains   ", "p": "pools without gains"}
    for k in forms:
        dev_ms, wall_ms = res[k]
        print("(%s) %s: stream time %.4f ms/step (median; CUDA events), host wall %.4f ms/step (median over rounds; "
              "rounds %.3f - %.3f), %d kernels per step (incl. the draws of picks and starts)" %
              (k, names[k], med(dev_ms), med(wall_ms), min(wall_ms), max(wall_ms), launches[k]))
    print("build: source_pool with targets %.1f ms, without %.1f ms (medians of 3, %d candidates): ss_pool_loudness "
          "%.3f ms per 30 s candidate" % (1e3 * with_t, 1e3 * without_t, len(spk_c) + len(noi_c), per_cand_ms))
    print("(g) == (p) x float32 gain on the same draws, bit for bit (stems)")
    for k in forms:
        plans[k][0].close()
        for p in pools[k]:
            p.close()


if __name__ == "__main__":
    main()
