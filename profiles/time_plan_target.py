"""Dereverberation targets in the training step: what it costs a plan's mixtures to also write every speaker's folded,
gained direct-path crop (Mixture(..., direct_out=...), k_mix_write<true>).

Workload: a pool of 32 bench.py configs[1] scenes (64 banked moving speakers, P = 40, C = 6, L = 4096, 30 s) with mono
level tables and direct sets of 40 taps, 32 banked static noises; 16 examples per step, each a random scene, its 2
speakers in random order and its noise, one 4 s crop drawn on the device (CropDraw, 101 tries, -40 dB), SIRs ~ U(-6, 6),
SNRs ~ U(10, 20), mono mixtures.  Both plans render the same direct stems (direct_taps = 40); (t) also writes the
targets, (n) does not.
  - Step time: (n) and (t) alternating, 8 rounds x 30 steps, CUDA events around each step: median, p10 and p90.
  - k_mix_write time per step: torch.profiler over 10 steps of each form, in a run of its own.
  - Extra bytes per step from shapes: per mixture, S direct stems read (S * C * T floats) and S * T floats written.
  - A check that (t) and (n) give the same stems, direct stems, mixtures and starts on the same draws.
Prints the card and its power limit."""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__)).rsplit(os.sep, 1)[0]
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from sonicsim_b200 import render  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U, SCENES, TRIES, TAPS = 4 * 16000, 16, 32, 101, 40
STEPS, ROUNDS, PROF_STEPS = 30, 8, 10


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(SCENES, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(9)
    spk_c = [render.MovingSource(to(x), R.rir_bank(to(h), direct_taps=TAPS), to(b), b) for x, h, b in items]
    noi_c = []
    for _ in range(SCENES):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        noi_c.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    spk_pool, noi_pool = R.source_pool(spk_c, levels="mono"), R.source_pool(noi_c)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)

    def plan(targets):
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        douts = [torch.empty((C, CROP), device=dev) if k < S else None for _ in range(U) for k in range(S + 1)]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk_pool, picks[e, k], (starts[e], CROP), TAPS) for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[e], (starts[e], CROP)))
        mix, sp, rms = (torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev),
                        torch.empty((U, S), device=dev))
        tgt = torch.empty((U, S, CROP), device=dev) if targets else None
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True, direct_out=tgt[e] if targets else None) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        p = R.plan_device(srcs, outs, douts, mixtures=mixes, draws=draws)
        return p, dict(outs=outs, douts=[d for d in douts if d is not None], mix=[mix], sp=[sp], rms=[rms],
                       starts=[starts], used=[used])

    plan_n, o_n = plan(False)
    plan_t, o_t = plan(True)

    def choose():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)
        u.uniform_()

    forms = (("n", plan_n), ("t", plan_t))
    for _ in range(3):
        for _, p in forms:
            choose()
            p.run()
    choose()
    plan_n.run()
    plan_t.run()
    torch.cuda.synchronize()
    for k in o_n:
        for a, b in zip(o_n[k], o_t[k]):
            assert torch.equal(a, b), k
    R.check_device_errors()
    launches = []
    for _, p in forms:
        R.reset_stats()
        p.run()
        launches.append(R.launch_count())
    assert plan_n.is_graph() and plan_t.is_graph()

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: [] for k, _ in forms}
    for _ in range(ROUNDS):
        for key, p in forms:
            torch.cuda.synchronize()
            for e0, e1 in ev:
                choose()
                e0.record()
                p.run()
                e1.record()
            torch.cuda.synchronize()
            res[key] += [e0.elapsed_time(e1) for e0, e1 in ev]
    R.check_device_errors()

    kern = {}
    for key, p in forms:
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(PROF_STEPS):
                choose()
                p.run()
            torch.cuda.synchronize()
        us = [e.device_time_total for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
              and "k_mix_write" in e.name]
        kern[key] = (sum(us) / 1e3 / PROF_STEPS, len(us) // PROF_STEPS)

    q = lambda v, p: float(np.percentile(v, p))                                             # noqa: E731
    print("workload: pool of %d scenes (bench.py configs[1], C = %d, direct_taps = %d), %d examples per step (%d "
          "speakers + 1 noise), %d-sample mono crops drawn on the device (%d tries); %d rounds x %d steps per form, "
          "alternating" % (SCENES, C, TAPS, U, S, CROP, TRIES, ROUNDS, STEPS))
    names = {"n": "no targets", "t": "with targets"}
    for (key, _), nl in zip(forms, launches):
        v = res[key]
        print("(%s) %s: step %.4f ms (median), p10 %.4f, p90 %.4f; k_mix_write %.4f ms per step (%d launch per "
              "step, profiled run); %d launches per run" % (key, names[key], q(v, 50), q(v, 10), q(v, 90), kern[key][0],
                                                            kern[key][1], nl))
    print("(t) / (n) median step time: %.4f; k_mix_write (t) - (n): %.4f ms" %
          (q(res["t"], 50) / q(res["n"], 50), kern["t"][0] - kern["n"][0]))
    rd, wr = 4 * U * S * C * CROP, 4 * U * S * CROP
    print("extra bytes per step from shapes: %d read (S direct stems of C x T floats per mixture) + %d written (S x T "
          "floats per mixture) = %.1f MB" % (rd, wr, (rd + wr) / 1e6))
    print("(t) == (n) on stems, direct stems, mix, speakers_out, rms_db, starts and used, bit for bit")
    for p in (plan_n, plan_t, spk_pool, noi_pool):
        p.close()


if __name__ == "__main__":
    main()
