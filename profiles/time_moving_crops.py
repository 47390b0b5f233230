"""Training crops that move every step: render_device with host starts against a plan whose starts live on the device.

Workload: bench.py's inputs (16 configs[1] utterances = 32 speakers, P = 40, C = 6, L = 4096, 30 s), every speaker from
an RIR bank, one 4 s crop per speaker per step, new random starts every step.
(a) render_device: the starts are drawn on the host and passed as ints, a new batch per step (validation, chunking,
    host block planning, descriptor upload and launches at every call);
(b) plan_device once, each window's start an element of a (32,) CUDA int32 tensor: a step is
    starts.copy_(torch.randint(...)) and plan.run() (one CUDA graph launch).
Per step: stream time (CUDA events around the step, median), host wall time (a run of steps back to back, ending in a
synchronise, divided by the steps) and the host time of the calls alone (median).  The two forms alternate.  Asserts in
the same run that every crop equals the slice of the full stem, bit for bit, on both forms.  Prints the card and its
power limit.  Informational: bench.py is unchanged."""
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
CROP, U = 4 * 16000, 16
STEPS, ROUNDS = 50, 8


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(U, 0)
    n = len(items)
    C, N = bench.CFG["C"], bench.CFG["N"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_x = [to(x) for x, _, _ in items]
    d_b = [to(b) for _, _, b in items]
    banks = [R.rir_bank(to(h)) for _, h, _ in items]
    srcs = [render.MovingSource(x, bk, b, bh) for x, bk, b, (_, _, bh) in zip(d_x, banks, d_b, items)]
    full = [torch.empty((C, N), device=dev) for _ in range(n)]
    R.render_device(srcs, full)

    rng = np.random.default_rng(7)
    outs_a = [torch.empty((C, CROP), device=dev) for _ in range(n)]

    def step_a():
        a = rng.integers(0, N - CROP + 1, n)
        R.render_device([s._replace(window=(int(v), CROP)) for s, v in zip(srcs, a)], outs_a)
        return a

    starts = torch.zeros(n, dtype=torch.int32, device=dev)
    outs_b = [torch.empty((C, CROP), device=dev) for _ in range(n)]
    plan = R.plan_device([s._replace(window=(starts[k], CROP)) for k, s in enumerate(srcs)], outs_b)

    def step_b():
        starts.copy_(torch.randint(0, N - CROP + 1, (n,), dtype=torch.int32, device=dev))
        plan.run()

    def check(outs, a):
        for k in range(n):
            assert torch.equal(outs[k], full[k][:, int(a[k]):int(a[k]) + CROP]), k

    for _ in range(5):                                   # warm-up, graph capture, then the bit checks
        step_a(); step_b()
    for _ in range(5):
        a = step_a()
        torch.cuda.synchronize()
        check(outs_a, a)
        step_b()
        a = starts.cpu().numpy()                         # (synchronises)
        check(outs_b, a)
    R.check_device_errors()
    launches = []
    for f in (step_a, step_b):
        c0 = R.launch_count()
        f()
        torch.cuda.synchronize()
        launches.append(R.launch_count() - c0)

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
    a_last = starts.cpu().numpy()
    check(outs_b, a_last)
    med = lambda v: float(np.median(v))
    spread = lambda v: "%.3f - %.3f" % (min(v), max(v))
    print("workload: %d speakers (bench.py configs[1], banked), one %d-sample crop each per step, new random starts "
          "every step; %d rounds x %d steps per form, alternating" % (n, CROP, ROUNDS, STEPS))
    for key, name, nl in (("a", "render_device, host starts", launches[0]),
                          ("b", "plan with device starts ", launches[1])):
        dev_ms, wall_ms, call_ms = res[key]
        print("(%s) %s: stream time %.4f ms/step (median; CUDA events), host wall %.4f ms/step (median over rounds; "
              "rounds %s), host calls %.4f ms/step (median), %d kernel launches per step" %
              (key, name, med(dev_ms), med(wall_ms), spread(wall_ms), med(call_ms), nl))
    print("crops == full stems sliced, bit for bit, on both forms")
    plan.close()
    for bk in banks:
        bk.close()


if __name__ == "__main__":
    main()
