"""The separation dataloader's training step with its random choices on the device: scenes, speakers, crops, mixtures.

Pool: 64 bench.py configs[1] utterances (128 banked moving speakers, P = 40, C = 6, L = 4096, 30 s) and one seeded banked
static noise per utterance (64).  Batch: 16 examples per step, each a random scene (`random.choice`, movingdatamodule.py
:57), its 2 speakers in random order (`random.sample`, :59) and its noise, one 4 s crop per example with a new start, SIRs
~ U(-6, 6), SNRs ~ U(10, 20), mono mixtures (mix (16, T), speakers (16, 2, T)) as movingdatamodule.py:56-126 returns them.
(a) scenes, speakers and starts drawn on the host, render_device of the chosen banked sources with those windows, then
    the dataloader's arithmetic as batched torch ops - the best route without pools;
(b) a plan of 48 pooled slots with mixtures, picks and starts drawn on the device: one graph launch per step;
(c) a plan over 16 fixed banked scenes with moving windows and mixtures (no pools), to isolate what pooling costs on
    the device (k_prepare reading its table from global memory, tables sized for the largest candidate).
Per step: stream time (CUDA events around the step, median), host wall time (a run of steps back to back, ending in a
synchronise, divided by the steps), the host time of the calls alone (median) and kernel launches (torch.profiler over
one step).  The forms alternate.  Asserts in the same run that (b)'s stems equal (a)'s bit for bit on the same draws.
Prints the card and its power limit.  Informational: bench.py is unchanged."""
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
from time_train_step import torch_mix  # noqa: E402
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
    spk_pool, noi_pool = R.source_pool(spk_c), R.source_pool(noi_c)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    starts = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)

    def stems():
        spk = torch.empty((U, S, C, CROP), device=dev)
        noi = torch.empty((U, 1, C, CROP), device=dev)
        outs = []
        for u in range(U):
            outs += [spk[u, k] for k in range(S)] + [noi[u, 0]]
        return spk, noi, outs

    def mixtures():
        mix, out, rms = torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev), \
            torch.empty((U, S), device=dev)
        return [render.Mixture(list(range((S + 1) * u, (S + 1) * u + S)), [(S + 1) * u + S], sirs[u], snr[u], mix[u],
                               out[u], rms[u], mono=True) for u in range(U)]

    # (a) host draws, render_device, torch arithmetic
    spk_a, noi_a, outs_a = stems()
    host_rng = np.random.default_rng(6)
    res_a = {}

    def srcs_a(sc, perm, st):
        srcs = []
        for u in range(U):
            srcs += [spk_c[S * sc[u] + perm[u, k]]._replace(window=(int(st[u]), CROP)) for k in range(S)]
            srcs.append(noi_c[sc[u]]._replace(window=(int(st[u]), CROP)))
        return srcs

    def step_a():
        sc = host_rng.integers(0, SCENES, U)
        perm = np.argsort(host_rng.random((U, S)), axis=1)
        st = host_rng.integers(0, N - CROP + 1, U)
        R.render_device(srcs_a(sc, perm, st), outs_a)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)
        res_a["mix"], res_a["spk"] = torch_mix(spk_a, noi_a, sirs, snr)

    # (b) pooled plan
    spk_b, noi_b, outs_b = stems()
    srcs_b = []
    for u in range(U):
        srcs_b += [render.Pooled(spk_pool, picks[u, k], (starts[u], CROP)) for k in range(S)]
        srcs_b.append(render.Pooled(noi_pool, scene[u], (starts[u], CROP)))
    plan_b = R.plan_device(srcs_b, outs_b, mixtures=mixtures())

    def step_b():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        starts.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)
        plan_b.run()

    # (c) fixed scenes with moving windows
    spk_c_, noi_c_, outs_c = stems()
    srcs_c = []
    for u in range(U):
        srcs_c += [spk_c[S * u + k]._replace(window=(starts[u], CROP)) for k in range(S)]
        srcs_c.append(noi_c[u]._replace(window=(starts[u], CROP)))
    plan_c = R.plan_device(srcs_c, outs_c, mixtures=mixtures())

    def step_c():
        starts.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)
        plan_c.run()

    def check_same_draws():
        """(b) and (a) on the same scenes, speaker orders and starts: the same stems, bit for bit."""
        sc = host_rng.integers(0, SCENES, U)
        perm = np.argsort(host_rng.random((U, S)), axis=1)
        st = host_rng.integers(0, N - CROP + 1, U)
        picks.copy_(torch.from_numpy((S * sc[:, None] + perm).astype(np.int32)))
        scene.copy_(torch.from_numpy(sc.astype(np.int32)))
        starts.copy_(torch.from_numpy(st.astype(np.int32)))
        plan_b.run()
        R.render_device(srcs_a(sc, perm, st), outs_a)
        torch.cuda.synchronize()
        assert torch.equal(spk_a, spk_b) and torch.equal(noi_a, noi_b)

    forms = (("a", step_a), ("b", step_b), ("c", step_c))
    for _ in range(5):                                   # warm-up and graph capture
        for _, f in forms:
            f()
    check_same_draws()
    R.check_device_errors()
    launches = []
    for _, f in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        launches.append(sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA))

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: ([], [], []) for k, _ in forms}
    for _ in range(ROUNDS):
        for key, f in forms:
            dev_ms, wall_ms, call_ms = res[key]
            torch.cuda.synchronize()
            calls = []
            t0 = time.perf_counter()
            for e0, e1 in ev:
                c0 = time.perf_counter()
                e0.record()
                f()
                e1.record()
                calls.append(time.perf_counter() - c0)
            torch.cuda.synchronize()
            wall_ms.append(1e3 * (time.perf_counter() - t0) / STEPS)
            dev_ms += [e0.elapsed_time(e1) for e0, e1 in ev]
            call_ms += [1e3 * c for c in calls]
    check_same_draws()
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    spread = lambda v: "%.3f - %.3f" % (min(v), max(v))                                     # noqa: E731
    print("workload: pool of %d scenes (bench.py configs[1], %d banked speakers, %d banked static noises); %d examples "
          "per step, each a random scene, its speakers in random order and its noise, one %d-sample mono crop, new "
          "SIRs and SNRs; %d rounds x %d steps per form, alternating" %
          (SCENES, S * SCENES, SCENES, U, CROP, ROUNDS, STEPS))
    names = {"a": "host draws + render_device + torch", "b": "pooled plan with mixtures         ",
             "c": "fixed scenes, moving windows      "}
    for (key, _), nl in zip(forms, launches):
        dev_ms, wall_ms, call_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median; CUDA events), host wall %.4f ms/step (median over rounds; "
              "rounds %s), host calls %.4f ms/step (median), %d kernels per step (incl. the draws)" %
              (key, names[key], med(dev_ms), med(wall_ms), spread(wall_ms), med(call_ms), nl))
    print("(b) == (a) on the same draws, bit for bit (stems)")
    plan_b.close()
    plan_c.close()
    spk_pool.close()
    noi_pool.close()


if __name__ == "__main__":
    main()
