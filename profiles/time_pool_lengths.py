"""A training step over a speaker pool whose RIR lengths differ, against the same speakers zero-padded to the longest L.

SonicSet gives every speaker of a scene its own RIR length (one generate_rir_combination call per speaker, SonicSet.py
:60-66), but the distribution of those lengths over real dumps is not known here.  This profile uses a SYNTHETIC spread:
32 bench.py configs[1]-shaped speakers (C = 6, P = 40, N = 480000) whose L is drawn uniformly from [1000, 16384] with a
seeded generator and then forced so that every K = ceil(L / 4096) in 1..4 occurs 8 times (taps past configs[1]'s 4096
are a seeded decaying tail), and 16 static noises with L = 4096.  Batch: 16 examples per step, 2 pooled speakers and 1
pooled noise each, one 4 s crop per example with a new start, mono mixtures (profiles/time_pool_step.py (b)).
(m) the speaker pool as is: every candidate renders with its own K;
(p) the same speakers with their RIRs zero-padded to the longest L: every candidate renders with K = 4.
Per form: stream time per step (CUDA events, median), host wall time per step (back-to-back steps ending in a
synchronise, median over rounds), kernels per step (torch.profiler over one step), and the speaker banks' bytes (exact,
from shapes: sum of P * C * K * 4096 * 8).  The forms alternate.  Both forms see the same draws; their stems agree to
float32 rounding (the max relative difference is printed).  Prints the card and its power limit."""
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
CROP, U, NSPK = 4 * 16000, 16, 32
STEPS, ROUNDS = 30, 6


def lengths(rng):
    L = rng.integers(1000, 16385, NSPK)
    for j in range(NSPK):                                # every K in 1..4, 8 times: the spread is named, not left to luck
        k = j % 4
        L[j] = min(max(L[j], 4096 * k + 1), 4096 * (k + 1))
    return [int(v) for v in L]


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(NSPK // 2, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(23)
    Ls = lengths(rng)
    Lmax = max(Ls)
    spk = {"m": [], "p": []}
    bank_bytes = {"m": 0, "p": 0}
    for j in range(NSPK):
        x, h, b = items[j // 2]
        L = Ls[j]
        hh = np.zeros(h.shape[:-1] + (L,), np.float32)
        hh[..., :min(L, 4096)] = h[..., :min(L, 4096)]
        if L > 4096:
            tail = rng.standard_normal(h.shape[:-1] + (L - 4096,)) * np.exp(-np.arange(L - 4096) / 3000.0)
            hh[..., 4096:] = (tail * 0.01 * float(np.abs(h).max())).astype(np.float32)
        hp = np.zeros(h.shape[:-1] + (Lmax,), np.float32)
        hp[..., :L] = hh
        P = h.shape[0]
        for key, rr in (("m", hh), ("p", hp)):
            spk[key].append(render.MovingSource(to(x), R.rir_bank(to(rr)), to(b), b))
            bank_bytes[key] += P * C * ((rr.shape[-1] + 4095) // 4096) * 4096 * 8
    noi = []
    for _ in range(U):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        noi.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    noi_pool = R.source_pool(noi)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    starts = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)
    pools, plans, outs = {}, {}, {}
    for key in ("m", "p"):
        pools[key] = R.source_pool(spk[key])
        srcs, o = [], []
        for u in range(U):
            srcs += [render.Pooled(pools[key], picks[u, k], (starts[u], CROP)) for k in range(S)]
            srcs.append(render.Pooled(noi_pool, scene[u], (starts[u], CROP)))
            o += [torch.empty((C, CROP), device=dev) for _ in range(S + 1)]
        mix, so_, rms = torch.empty((U, CROP), device=dev), torch.empty((U, S, CROP), device=dev), \
            torch.empty((U, S), device=dev)
        mixtures = [render.Mixture(list(range((S + 1) * u, (S + 1) * u + S)), [(S + 1) * u + S], sirs[u], snr[u],
                                   mix[u], so_[u], rms[u], mono=True) for u in range(U)]
        plans[key], outs[key] = R.plan_device(srcs, o, mixtures=mixtures), o

    def draw():
        picks.copy_(torch.randint(0, NSPK, (U, S), device=dev, dtype=torch.int32))
        scene.copy_(torch.randint(0, U, (U,), device=dev, dtype=torch.int32))
        starts.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    forms = {k: (lambda k=k: (draw(), plans[k].run())) for k in ("m", "p")}
    for _ in range(5):                                   # warm-up and graph capture
        for f in forms.values():
            f()
    draw()
    for k in ("m", "p"):
        plans[k].run()
    torch.cuda.synchronize()
    rel = max(float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30) for a, b in zip(outs["m"], outs["p"]))
    R.check_device_errors()
    launches = {}
    for key, f in forms.items():
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        launches[key] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: ([], []) for k in forms}
    for _ in range(ROUNDS):
        for key, f in forms.items():
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
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    ks = [(L + 4095) // 4096 for L in Ls]
    print("workload: %d configs[1]-shaped speakers, synthetic L spread %s (K counts %s), longest L %d; %d static noises "
          "(L = 4096); %d examples per step (2 pooled speakers + 1 pooled noise, %d-sample mono crops, mixtures); "
          "%d rounds x %d steps per form, alternating" %
          (NSPK, sorted(Ls), {k: ks.count(k) for k in sorted(set(ks))}, Lmax, U, U, CROP, ROUNDS, STEPS))
    names = {"m": "mixed-length pool  ", "p": "padded to longest L"}
    for key in forms:
        dev_ms, wall_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median; CUDA events), host wall %.4f ms/step (median over rounds; "
              "rounds %.3f - %.3f), %d kernels per step, speaker banks %d bytes, pool %d bytes" %
              (key, names[key], med(dev_ms), med(wall_ms), min(wall_ms), max(wall_ms), launches[key],
               bank_bytes[key], pools[key].nbytes))
    print("(m) vs (p) on the same draws: max |difference| / max |stem| = %.3g" % rel)
    for k in ("m", "p"):
        plans[k].close()
        pools[k].close()
    noi_pool.close()


if __name__ == "__main__":
    main()
