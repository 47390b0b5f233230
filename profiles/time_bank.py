"""RIR spectrum banks (ss_bank): bench.py's configs[1] pass with raw RIRs against the same pass from banks.

(a) device path: bench.py's inputs (16 utterances = 32 speakers, P = 40, C = 6, L = 4096, 30 s), one plan, raw vs banked;
(b) the same pass through plan_host (pinned buffers), next to its copy-only floor at the banked byte count (dry in, stems
    out, no RIRs);
(c) the same 32 speakers as one 4 s window each, one plan, raw vs banked.
Times with CUDA events, warmed up, the two forms alternating, median of the repetitions; asserts in the same run that
banked and raw outputs are bit-identical; prints the card, the transform counts and H2D bytes computed from the shapes,
and the bank creation time per speaker.  Informational: bench.py itself is unchanged."""
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
from time_window import card, median_ms, transforms  # noqa: E402

dev = torch.device("cuda", 0)
SR, CROP, U = 16000, 4 * 16000, 16


def timed(fn, runs):
    def f():
        for _ in range(runs):
            fn()
    return f


def main():
    R = render.Renderer(0)
    print("device:", card())
    items = bench.make_inputs(U, 0)
    n = len(items)
    P, C, L, N = bench.CFG["P"], bench.CFG["C"], bench.CFG["L"], bench.CFG["N"]
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    d_x = [to(x) for x, _, _ in items]
    d_h = [to(h) for _, h, _ in items]
    d_b = [to(b) for _, _, b in items]

    # bank creation: per speaker, from device memory (on the current stream) and from host memory
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t_dev = []
    banks = []
    for k in range(n):
        e0.record()
        bk = R.rir_bank(d_h[k])
        e1.record()
        torch.cuda.synchronize()
        t_dev.append(e0.elapsed_time(e1))
        banks.append(bk)
    # from host memory (synchronous: wall time), pageable and pinned, and ss_bank_destroy on its own
    t_host, t_pin, t_free = [], [], []
    for k in range(8):
        t0 = time.perf_counter()
        bk = R.rir_bank(items[k][1])
        t1 = time.perf_counter()
        bk.close()
        t2 = time.perf_counter()
        bp = R.rir_bank(torch.from_numpy(items[k][1]).pin_memory().numpy())
        t3 = time.perf_counter()
        bp.close()
        t_host.append(1e3 * (t1 - t0)); t_free.append(1e3 * (t2 - t1)); t_pin.append(1e3 * (t3 - t2))
    bank_b = banks[0].nbytes
    med = lambda v: float(np.median(v))
    print("bank: %.3f MB per speaker (%d speakers: %.1f MB); creation per speaker: %.3f ms from device memory "
          "(median of %d; first %.3f); from host memory (%.2f MB): %.3f ms pageable, %.3f ms pinned (median of 8, "
          "first %.3f / %.3f); ss_bank_destroy %.3f ms (median of 8)" %
          (bank_b / 1e6, n, n * bank_b / 1e6, med(t_dev[1:]), n - 1, t_dev[0], P * C * L * 4 / 1e6, med(t_host),
           med(t_pin), t_host[0], t_pin[0], med(t_free)))
    tr = np.sum([transforms(x, h, b, None) for x, h, b in items], axis=0)
    print("transforms per pass (RIR pairs, dry pairs, inverse): raw %s, banked %s" % (tuple(tr), (0,) + tuple(tr[1:])))
    rir_b, dry_b, out_b = n * P * C * L * 4, n * N * 4, n * C * N * 4
    print("host path bytes per pass: H2D raw %.1f MB (RIRs %.1f MB), banked %.1f MB; D2H %.1f MB" %
          ((rir_b + dry_b + n * P * 4) / 1e6, rir_b / 1e6, (dry_b + n * P * 4) / 1e6, out_b / 1e6))

    # (a) device pass, one plan each
    o_raw = [torch.empty((C, N), device=dev) for _ in range(n)]
    o_bank = [torch.empty((C, N), device=dev) for _ in range(n)]
    p_raw = R.plan_device([render.MovingSource(x, h, b, bh) for x, h, b, (_, _, bh) in zip(d_x, d_h, d_b, items)], o_raw)
    p_bank = R.plan_device([render.MovingSource(x, bk, b, bh) for x, bk, b, (_, _, bh) in zip(d_x, banks, d_b, items)],
                           o_bank)
    for _ in range(5):
        p_raw.run(); p_bank.run()
    torch.cuda.synchronize()
    for a, b in zip(o_raw, o_bank):
        assert torch.equal(a, b)
    ra, ba = median_ms([timed(p_raw.run, 10), timed(p_bank.run, 10)], 30)
    print("(a) device pass, %d speakers, one plan: raw %.3f ms, banked %.3f ms per pass (%+.1f %%)" %
          (n, ra / 10, ba / 10, 100 * (ba - ra) / ra))

    # (b) host pass through plan_host, pinned buffers
    hx = [torch.from_numpy(x).pin_memory() for x, _, _ in items]
    hh = [torch.from_numpy(h).pin_memory() for _, h, _ in items]
    ho_raw = [torch.empty((C, N)).pin_memory() for _ in range(n)]
    ho_bank = [torch.empty((C, N)).pin_memory() for _ in range(n)]
    hp_raw = R.plan_host([render.MovingSource(x.numpy(), h.numpy(), b) for x, h, (_, _, b) in zip(hx, hh, items)],
                         [o.numpy() for o in ho_raw])
    hp_bank = R.plan_host([render.MovingSource(x.numpy(), bk, b) for x, bk, (_, _, b) in zip(hx, banks, items)],
                          [o.numpy() for o in ho_bank])
    hp_raw.run(); hp_bank.run()
    for a, b in zip(ho_raw, ho_bank):
        assert torch.equal(a, b)
    s_in, s_out = torch.cuda.Stream(dev), torch.cuda.Stream(dev)

    def copy_floor():                      # the banked pass's bytes: dry in, stems out, on two streams
        with torch.cuda.stream(s_in):
            for h_, d_ in zip(hx, d_x):
                d_.copy_(h_, non_blocking=True)
        with torch.cuda.stream(s_out):
            for h_, d_ in zip(ho_bank, o_bank):
                h_.copy_(d_, non_blocking=True)
        torch.cuda.current_stream().wait_stream(s_in)
        torch.cuda.current_stream().wait_stream(s_out)
    copy_floor()
    torch.cuda.synchronize()
    rb_, bb_, fl = median_ms([hp_raw.run, hp_bank.run, copy_floor], 12)
    print("(b) host pass (plan_host), %d speakers: raw %.2f ms, banked %.2f ms (%+.1f %%); copy-only floor at the "
          "banked bytes %.2f ms" % (n, rb_, bb_, 100 * (bb_ - rb_) / rb_, fl))

    # (c) one 4 s window per speaker
    rng = np.random.default_rng(11)
    wins = [(int(rng.integers(0, N - CROP + 1)), CROP) for _ in range(n)]
    w_raw = [torch.empty((C, CROP), device=dev) for _ in range(n)]
    w_bank = [torch.empty((C, CROP), device=dev) for _ in range(n)]
    pw_raw = R.plan_device([render.MovingSource(x, h, b, bh, window=w) for x, h, b, (_, _, bh), w in
                            zip(d_x, d_h, d_b, items, wins)], w_raw)
    pw_bank = R.plan_device([render.MovingSource(x, bk, b, bh, window=w) for x, bk, b, (_, _, bh), w in
                             zip(d_x, banks, d_b, items, wins)], w_bank)
    for _ in range(5):
        pw_raw.run(); pw_bank.run()
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(zip(w_raw, w_bank)):
        assert torch.equal(a, b)
        assert torch.equal(b, o_raw[k][:, wins[k][0]:wins[k][0] + CROP])
    tw = np.sum([transforms(x, h, b, w) for (x, h, b), w in zip(items, wins)], axis=0)
    rc, bc = median_ms([timed(pw_raw.run, 10), timed(pw_bank.run, 10)], 30)
    print("(c) %d x 4 s windows, one plan: transforms raw %s, banked %s; raw %.4f ms, banked %.4f ms per pass "
          "(%+.1f %%)" % (n, tuple(tw), (0,) + tuple(tw[1:]), rc / 10, bc / 10, 100 * (bc - rc) / rc))
    print("banked == raw, bit for bit, in (a), (b) and (c)")
    for p in (p_raw, p_bank, pw_raw, pw_bank):
        p.close()
    for bk in banks:
        bk.close()


if __name__ == "__main__":
    main()
