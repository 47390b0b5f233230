"""The separation dataloader's training step on the device: crops, then mixtures, every step.

Workload: bench.py's inputs (16 configs[1] utterances = 32 speakers, P = 40, C = 6, L = 4096, 30 s), every speaker from
an RIR bank, plus one seeded static noise source per utterance (C = 6, L = 4096, banked).  Every step takes one 4 s crop
of each utterance (its two speakers and its noise share one device start) with new starts, SIRs ~ U(-6, 6) and SNRs ~
U(10, 20), and returns (mix (16, T), speakers (16, 2, T)) with the dataloader's defaults (is_mono: channel mean first),
as movingdatamodule.py:56-126 does per example.
(a) the crop plan (plan_device with device starts), then the dataloader's arithmetic as batched torch ops on the
    device - the best a caller could write without mixtures in plans;
(b) the same plan with one Mixture per utterance: one graph launch per step.
Per step: stream time (CUDA events around the step, median), host wall time (a run of steps back to back, ending in a
synchronise, divided by the steps), the host time of the calls alone (median) and kernel launches (torch.profiler over
one step).  The two forms alternate.  Asserts in the same run that (b)'s outputs equal ss_mix_dev on (b)'s own crops,
folded in the stated order, bit for bit; reports the largest difference between (a) and (b) in float32 ulps of the batch's largest value.  Prints
the card and its power limit.  Informational: bench.py is unchanged."""
import ctypes
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from sonicsim_b200 import _lib, render  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U = 4 * 16000, 16
STEPS, ROUNDS = 50, 8


def torch_mix(spk, noi, sirs, snr):
    """movingdatamodule.py:62-63, 76-77, 104-124 batched: spk (B, S, C, T), noi (B, M, C, T), sirs (B, S - 1), snr (B,)
    -> mix (B, T), speakers after their gains (B, S, T)."""
    s, n = spk.mean(dim=2), noi.mean(dim=2)
    db = lambda x: 10 * torch.log10(torch.clamp((x ** 2).mean(dim=-1), min=1e-20))          # noqa: E731
    e = db(s)
    gain = torch.clamp(e[:, :1] - e[:, 1:] - sirs, max=40.0)
    g = torch.cat([torch.ones_like(gain[:, :1]), 10 ** (gain / 20)], dim=1)
    out = s * g[..., None]
    speech = out.sum(dim=1)
    noise = n.sum(dim=1)
    gn = 10 ** (torch.clamp(db(speech) - db(noise) - snr, max=40.0) / 20)
    return speech + noise * gn[:, None], out


def fold(a):
    acc = a[0].copy()
    for c in range(1, a.shape[0]):
        acc = acc + a[c]
    return acc / np.float32(a.shape[0])


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(U, 0)
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                        # noqa: E731
    rng = np.random.default_rng(5)
    spk_srcs = [render.MovingSource(to(x), R.rir_bank(to(h)), to(b), b) for x, h, b in items]
    noi_srcs = []
    for u in range(U):
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        noi_srcs.append(render.StaticSource(to(x), R.rir_bank(to(h))))
    starts = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)
    srcs = []
    for u in range(U):
        srcs += [spk_srcs[S * u + k]._replace(window=(starts[u], CROP)) for k in range(S)]
        srcs.append(noi_srcs[u]._replace(window=(starts[u], CROP)))

    def stems():
        spk = torch.empty((U, S, C, CROP), device=dev)
        noi = torch.empty((U, 1, C, CROP), device=dev)
        outs = []
        for u in range(U):
            outs += [spk[u, k] for k in range(S)] + [noi[u, 0]]
        return spk, noi, outs

    spk_a, noi_a, outs_a = stems()
    plan_a = R.plan_device(srcs, outs_a)
    spk_b, noi_b, outs_b = stems()
    mix_b = torch.empty((U, CROP), device=dev)
    out_b = torch.empty((U, S, CROP), device=dev)
    rms_b = torch.empty((U, S), device=dev)
    mixtures = [render.Mixture(list(range((S + 1) * u, (S + 1) * u + S)), [(S + 1) * u + S], sirs[u], snr[u],
                               mix_b[u], out_b[u], rms_b[u], mono=True) for u in range(U)]
    plan_b = R.plan_device(srcs, outs_b, mixtures=mixtures)
    res_a = {}

    def draw():
        starts.copy_(torch.randint(0, N - CROP + 1, (U,), dtype=torch.int32, device=dev))
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)

    def step_a():
        draw()
        plan_a.run()
        res_a["mix"], res_a["spk"] = torch_mix(spk_a, noi_a, sirs, snr)

    def step_b():
        draw()
        plan_b.run()

    def check_b():
        """(b)'s outputs against ss_mix_dev on (b)'s own crops, folded in NumPy: bit for bit."""
        torch.cuda.synchronize()
        sp, no = spk_b.cpu().numpy(), noi_b.cpu().numpy()
        fs = torch.from_numpy(np.stack([np.stack([fold(sp[u, k]) for k in range(S)]) for u in range(U)])).to(dev)
        fn = torch.from_numpy(np.stack([fold(no[u, 0]) for u in range(U)])).to(dev)
        mix = torch.empty((U, CROP), device=dev)
        scr = torch.empty((U, int(R.lib.ss_mix_scratch_doubles())), dtype=torch.float64, device=dev)
        its = (_lib.SsMixItem * U)()
        sn = snr.cpu().numpy()
        for u in range(U):
            its[u] = _lib.SsMixItem(speakers=fs[u].data_ptr(), noises=fn[u].data_ptr(), sirs=sirs[u].data_ptr(),
                                    mix=mix[u].data_ptr(), speakers_out=fs[u].data_ptr(), scratch=scr[u].data_ptr(),
                                    E=CROP, S=S, M=1, snr=float(sn[u]))
        _lib.check(R.lib.ss_mix_dev(R.ctx, its, U, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
        torch.cuda.synchronize()
        assert torch.equal(mix, mix_b) and torch.equal(fs, out_b)

    for _ in range(5):                                   # warm-up, graph capture, then the checks
        step_a(); step_b()
    for _ in range(3):
        step_b()
        check_b()
    # (a) against (b) on the same starts, SIRs and SNRs
    draw()
    plan_a.run()
    plan_b.run()
    ma, sa = torch_mix(spk_a, noi_a, sirs, snr)
    torch.cuda.synchronize()
    # largest |a - b| in float32 ulps of the largest |b| of the batch (element-wise ulps are unbounded near zero)
    ulp = lambda a, b: float((a - b).abs().max() / (2.0 ** -23 * 2.0 ** torch.floor(torch.log2(b.abs().max()))))  # noqa: E731
    d_mix, d_spk = ulp(ma, mix_b), ulp(sa, out_b)
    R.check_device_errors()
    launches = []
    for f in (step_a, step_b):
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        launches.append(sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA))

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {"a": ([], [], []), "b": ([], [], [])}
    for _ in range(ROUNDS):
        for key, f in (("a", step_a), ("b", step_b)):
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
    check_b()
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    spread = lambda v: "%.3f - %.3f" % (min(v), max(v))                                     # noqa: E731
    print("workload: %d utterances (bench.py configs[1], banked speakers) + one banked static noise each, one "
          "%d-sample mono crop per utterance per step, new starts, SIRs and SNRs every step; %d rounds x %d steps "
          "per form, alternating" % (U, CROP, ROUNDS, STEPS))
    for key, name, nl in (("a", "crop plan + torch arithmetic", launches[0]),
                          ("b", "plan with mixtures          ", launches[1])):
        dev_ms, wall_ms, call_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median; CUDA events), host wall %.4f ms/step (median over rounds; "
              "rounds %s), host calls %.4f ms/step (median), %d kernels per step (incl. the draws)" %
              (key, name, med(dev_ms), med(wall_ms), spread(wall_ms), med(call_ms), nl))
    print("(b) == ss_mix_dev on its own crops, bit for bit; largest difference (a) vs (b), in float32 ulps of the batch's "
          "largest value: mix %.2f, speakers %.2f" % (d_mix, d_spk))
    plan_a.close()
    plan_b.close()


if __name__ == "__main__":
    main()
