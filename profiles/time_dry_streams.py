"""Dry streams in the training step: what it costs to lay out each speaker's dry stream at every run from a 16-bit
utterance pool (render.DryStream) instead of dry-picking prebuilt 60 s streams from a 16-bit pool (render.DryPick).

Workload of time_compact_dry_pool.py (DESIGN section 6): a pool of 64 bench.py configs[1] scenes (128 banked moving
speakers, P = 40, C = 6, L = 4096, 30 s) and 64 banked static noises in device memory; 16 examples per step, each a
random scene, its 2 speakers in random order and its noise, one 4 s mono crop, SIRs ~ U(-6, 6), SNRs ~ U(10, 20), one
CropDraw per example (tries = 101, threshold -40 dB) over the dry tables: 32 speaker crops per step.  Forms,
alternating round by round:
(id) dry picks from 256 prebuilt 60 s streams in a 16-bit device pool;  (sd) layouts over a 16-bit device pool of
     2000 utterances of 2 to 20 s (dry.long_audio_layouts for 60 s streams, m = 32);
(ih) as (id), the pool in pinned host memory;                            (sh) as (sd), the pool in pinned host memory.
The prebuilt streams are laid out by the same rule from the same utterances.  Per step: stream time (CUDA events around
the step, median), kernels per step and the k_stage and k_draw times (torch.profiler, separate steps), dry samples
staged per run; and the stream time of dry.long_audio_layouts refreshing 32 layouts, on its own.  Then the time and
peak memory of long_audio_layouts over a LibriSpeech-sized corpus, with and without max_selected (layout_cost).  Prints
the card and its power limit."""
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import bench  # noqa: E402  (its input generator only)
from sonicsim_b200 import dry, render  # noqa: E402
from time_host_dry_pool import kernel_ms  # noqa: E402
from time_window import card  # noqa: E402

dev = torch.device("cuda", 0)
CROP, U, SCENES, TRIES, RATE = 4 * 16000, 16, 64, 101, 16000
N_UTT, N_STREAM, TOTAL, MM = 2000, 256, 60 * 16000, 32
STEPS, ROUNDS = 30, 8
KB = 4096
FORMS = ("id", "sd", "ih", "sh")


def read_span(N, K, ws):
    """Dry samples k_stage writes for one staged slot: whole groups of 4 around stage_set's [xa, xb)."""
    xa, xb = max(ws - (K + 2) * KB, 0), min(ws + CROP + 2 * KB, N)
    return ((xb + 3) & ~3) - (xa & ~3)


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
    utts = [np.clip(np.round(rng.standard_normal(int(rng.integers(2 * RATE, 20 * RATE))) * 3000 *
                             rng.uniform(0.1, 1.0)), -32768, 32767).astype(np.int16) for _ in range(N_UTT)]
    lengths = torch.tensor([u.size for u in utts])
    g = torch.Generator().manual_seed(1)
    li, lo = dry.long_audio_layouts(lengths, TOTAL, MM, N_STREAM, generator=g)
    streams = []
    for a, o in zip(li.numpy(), lo.numpy()):
        k = np.zeros(TOTAL, np.int16)
        for i, p in zip(a, o):
            if i >= 0:
                k[p:p + utts[i].size] = utts[i]
        streams.append(k)
    torch.cuda.synchronize()
    pools = {"id": R.dry_pool(streams, levels=True, dtype="int16"),
             "sd": R.dry_pool(utts, levels=True, dtype="int16"),
             "ih": R.dry_pool(streams, levels=True, host=True, dtype="int16"),
             "sh": R.dry_pool(utts, levels=True, host=True, dtype="int16")}
    spk, noi = R.source_pool(spk_c), R.source_pool(noi_c)
    lengths_dev = lengths.to(dev)

    picks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    dpicks = torch.zeros((U, S), dtype=torch.int32, device=dev)
    ids = torch.full((U, S, MM), -1, dtype=torch.int32, device=dev)
    offs = torch.full((U, S, MM), -1, dtype=torch.int32, device=dev)
    scene = torch.zeros(U, dtype=torch.int32, device=dev)
    sirs = torch.zeros((U, S - 1), device=dev)
    snr = torch.zeros((U,), device=dev)
    u = torch.zeros((U, TRIES), dtype=torch.float64, device=dev)
    gen = torch.Generator(device=dev)
    gen.manual_seed(2)

    def plan(key):
        dp = pools[key]
        starts = torch.zeros(U, dtype=torch.int32, device=dev)
        used = torch.zeros(U, dtype=torch.int32, device=dev)
        outs = [torch.empty((C, CROP), device=dev) for _ in range(U * (S + 1))]
        srcs = []
        for e in range(U):
            srcs += [render.Pooled(spk, picks[e, k], (starts[e], CROP), 0,
                                   render.DryStream(dp, ids[e, k], offs[e, k]) if key[0] == "s"
                                   else render.DryPick(dp, dpicks[e, k])) for k in range(S)]
            srcs.append(render.Pooled(noi, scene[e], (starts[e], CROP)))
        mix = torch.empty((U, CROP), device=dev)
        sp, rms = torch.empty((U, S, CROP), device=dev), torch.empty((U, S), device=dev)
        mixes = [render.Mixture(list(range((S + 1) * e, (S + 1) * e + S)), [(S + 1) * e + S], sirs[e], snr[e], mix[e],
                                sp[e], rms[e], mono=True) for e in range(U)]
        draws = [render.CropDraw(starts[e], list(range((S + 1) * e, (S + 1) * e + S)), u[e], used[e])
                 for e in range(U)]
        return R.plan_device(srcs, outs, mixtures=mixes, draws=draws), starts

    plans = {k: plan(k) for k in FORMS}

    def layouts():
        a, o = dry.long_audio_layouts(lengths_dev, TOTAL, MM, U * S, generator=gen)
        ids.copy_(a.view(U, S, MM))
        offs.copy_(o.view(U, S, MM))

    def choose():
        sc = torch.randint(0, SCENES, (U,), device=dev, dtype=torch.int32)
        picks.copy_(S * sc[:, None] + torch.rand(U, S, device=dev).argsort(1).int())
        scene.copy_(sc)
        sirs.uniform_(-6, 6)
        snr.uniform_(10, 20)
        dpicks.random_(0, N_STREAM)
        u.uniform_()

    layouts()

    def stepper(key):
        def f():
            choose()
            plans[key][0].run()
        return f

    forms = [(k, stepper(k)) for k in FORMS]
    for _ in range(3):
        for _, f in forms:
            f()
    torch.cuda.synchronize()
    R.check_device_errors()
    launches, stage_ms, draw_ms = {}, {}, {}
    for key, f in forms:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                f()
            torch.cuda.synchronize()
        launches[key] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA) / 5
        stage_ms[key] = kernel_ms(prof, "k_stage") / 5
        draw_ms[key] = kernel_ms(prof, "k_draw") / 5
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            layouts()
        torch.cuda.synchronize()
    lay_kernels = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA) / 5
    st = plans["id"][1].cpu().numpy()
    samples = sum(read_span(N, 1, int(st[e])) for e in range(U) for _ in range(S))

    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(STEPS)]
    res = {k: [] for k, _ in forms}
    lay = []
    for _ in range(ROUNDS):
        for key, f in forms:
            torch.cuda.synchronize()
            for e0, e1 in ev:
                e0.record()
                f()
                e1.record()
            torch.cuda.synchronize()
            res[key] += [e0.elapsed_time(e1) for e0, e1 in ev]
        for e0, e1 in ev:
            e0.record()
            layouts()
            e1.record()
        torch.cuda.synchronize()
        lay += [e0.elapsed_time(e1) for e0, e1 in ev]
    R.check_device_errors()
    med = lambda v: float(np.median(v))                                                     # noqa: E731
    print("workload: time_compact_dry_pool.py's step: pool of %d scenes, %d examples per step (%d speaker crops of %d "
          "samples), start draws (101 tries) over the dry tables; %d prebuilt %d s streams or %d utterances of 2-20 s "
          "(layouts of m = %d); %d rounds x %d steps per form, alternating" %
          (SCENES, U, U * S, CROP, N_STREAM, TOTAL // RATE, N_UTT, MM, ROUNDS, STEPS))
    for k in FORMS:
        print("dry pool (%s): nbytes %.1f MB, host_nbytes %.1f MB" %
              (k, pools[k].nbytes / 1e6, pools[k].host_nbytes / 1e6))
    names = {"id": "prebuilt streams, device ", "sd": "layouts, device          ",
             "ih": "prebuilt streams, host   ", "sh": "layouts, host            "}
    for key, _ in forms:
        v = res[key]
        rm = [med(v[i * STEPS:(i + 1) * STEPS]) for i in range(ROUNDS)]
        print("(%s) %s: stream time %.4f ms/step (median; round medians %.4f - %.4f), %d kernels per step, k_stage "
              "%.4f ms/step, k_draw %.4f ms/step (profiled), k_stage writes %.2f MB/run (%d dry samples x 4 B)" %
              (key, names[key], med(v), min(rm), max(rm), launches[key], stage_ms[key], draw_ms[key], samples * 4 / 1e6,
               samples))
    for a, b in (("sd", "id"), ("sh", "ih")):
        print("(%s) - (%s) stream time: %+.4f ms/step, ratio %.4f" % (a, b, med(res[a]) - med(res[b]),
                                                                       med(res[a]) / med(res[b])))
    print("dry.long_audio_layouts, %d layouts of m = %d over %d utterances: %.4f ms/step (stream time, median), "
          "%d kernels" % (U * S, MM, N_UTT, med(lay), lay_kernels))
    for p, _ in plans.values():
        p.close()
    for p in list(pools.values()) + [spk, noi]:
        p.close()
    layout_cost()


def layout_cost():
    """dry.long_audio_layouts over a LibriSpeech-sized corpus (n = 2.8e5 utterances of 1 to 35 s, lengths on the
    device), 128 layouts of m = 32 for 60 s streams: stream time (median of 20 calls after 3) and peak bytes that torch
    allocates in the call, sorting every utterance and with max_selected = long_audio_max_selected."""
    n, count = 280000, 128
    g = torch.Generator(device=dev)
    g.manual_seed(3)
    lengths = torch.randint(RATE, 35 * RATE + 1, (n,), device=dev, generator=g)
    bound = dry.long_audio_max_selected(lengths, TOTAL)
    for label, ms in (("every utterance sorted", None), ("max_selected = %d" % bound, bound)):
        for _ in range(3):
            dry.long_audio_layouts(lengths, TOTAL, MM, count, generator=g, max_selected=ms)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        times = []
        for _ in range(20):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            dry.long_audio_layouts(lengths, TOTAL, MM, count, generator=g, max_selected=ms)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        peak = torch.cuda.max_memory_allocated() - base
        print("dry.long_audio_layouts, %d layouts of m = %d over n = %d utterances, %s: %.4f ms/call (stream time, "
              "median), peak %.1f MB allocated (%.1f B per row and utterance)" %
              (count, MM, n, label, float(np.median(times)), peak / 1e6, peak / (count * n)))


if __name__ == "__main__":
    t0 = time.perf_counter()
    main()
    print("total %.1f s" % (time.perf_counter() - t0))
