"""Training crops: full stems against 4 s windows (ss_source.win_start / win_len), device and host path.

Times with CUDA events, the two forms alternating, median of the repetitions; asserts in the same run that every window
equals the slice of the full render, bit for bit; prints the forward / inverse transform counts computed from the
shapes (blocks from ss_debug_plan).  Informational: bench.py's line is configs[1] without windows."""
import ctypes
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sonicsim_oracle as so
from sonicsim_b200 import _lib, render

R = None                                               # render.Renderer(0), made in __main__
dev = torch.device("cuda", 0)
SR, CROP = 16000, 4 * 16000


def card():
    props = torch.cuda.get_device_properties(0)
    limit = "unknown"
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        if q:
            limit = q[0]
    except (OSError, subprocess.SubprocessError):
        pass
    return "%s, power limit %s" % (props.name, limit)


def scene(rng, n_moving, n_static, N, P, C, L):
    """Host arrays of one scene: [(x, h (P, C, L), bounds)] + [(x, h (C, L), None)]."""
    out = []
    for _ in range(n_moving):
        x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
        out.append((x, h, render.trajectory_bounds(pos, N)))
    for _ in range(n_static):
        out.append((so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, L)[0], None))
    return out


def sources(stems, wins=None, device=False):
    t = (lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)) if device else (lambda a: a)
    res = []
    for k, (x, h, b) in enumerate(stems):
        win = None if wins is None else wins[k]
        if b is None:
            res.append(render.StaticSource(t(x), t(h), window=win))
        else:
            res.append(render.MovingSource(t(x), t(h), t(b), b if device else None, window=win))
    return res


def transforms(x, h, b, win):
    """(RIR pair transforms, dry-window pair transforms, inverse transforms) from the shapes: the blocks of the plan
    (ss_debug_plan) and, for a window, the rows and blocks its read set covers."""
    N = x.shape[0]
    P, C, L = (1,) + h.shape if b is None else h.shape
    K = (L + 4095) // 4096
    bb = np.ascontiguousarray(b if b is not None else [0], np.int32)
    it = _lib.SsSource(x=1, rir=1, out=1, bounds=bb.ctypes.data if b is not None else None, N=N, P=P, C=C, L=L,
                       mode=_lib.SS_MOVING_BOUNDS if b is not None else _lib.SS_STATIC,
                       bounds_host=bb.ctypes.data if b is not None else None)
    cap = (N + 4095) // 4096 + P
    full = np.zeros((cap, 4), np.int32)
    al = ctypes.c_int32()
    nf = _lib.load().ss_debug_plan(ctypes.byref(it), full.ctypes.data, cap, ctypes.byref(al))
    full = full[:nf]
    per = C if b is not None else (C + 1) // 2
    inv = lambda blocks: sum(per * (1 if al.value or b is None else (blk[3] - blk[2] + 2) // 2) for blk in blocks)
    if win is None:
        return (P * C * K + 1) // 2, (nf + 1) // 2, inv(full)
    a, n = win
    keep = np.nonzero((full[:, 0] < a + n) & (full[:, 0] + full[:, 1] > a))[0]
    k0, k1 = keep[0], keep[-1] + 1
    g0, g1 = max(0, k0 - (K - 1)) & ~1, min(nf, (k1 + 1) & ~1)
    if b is None:
        pa, pb = 0, 0
    elif al.value:
        pa, pb = full[k0, 2], full[k1 - 1, 3]
    else:
        seg = lambda s: min(int(np.searchsorted(b[1:], s, side="right")), P - 2)
        pa, pb = seg(full[k0, 0]), seg(full[k1 - 1, 0] + full[k1 - 1, 1] - 1) + 1
    ck = C * K
    r0, r1 = (pa * ck) & ~1, min(P * ck, ((pb + 1) * ck + 1) & ~1)
    blocks = full[k0:k1].copy()
    if not al.value and b is not None:                 # grid blocks: positions from the bounds
        for blk in blocks:
            blk[2] = min(int(np.searchsorted(b[1:], blk[0], side="right")), P - 2)
            blk[3] = min(int(np.searchsorted(b[1:], blk[0] + blk[1] - 1, side="right")), P - 2) + 1
    return (r1 - r0 + 1) // 2, (g1 - g0 + 1) // 2, inv(blocks)


def median_ms(fns, reps):
    """Median ms of each fn over `reps` rounds, the fns alternating within a round."""
    t = [[] for _ in fns]
    for _ in range(reps):
        for k, f in enumerate(fns):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            f()
            e1.record()
            torch.cuda.synchronize()
            t[k].append(e0.elapsed_time(e1))
    return [float(np.median(v)) for v in t]


def case(title, stems, n_crops, rng, reps=20):
    N = stems[0][0].shape[0]
    wins = [(int(rng.integers(0, N - CROP + 1)), CROP) for _ in range(n_crops * len(stems))]
    crop_stems = [stems[k % len(stems)] for k in range(len(wins))]
    # device path
    full_src = sources(stems, device=True)
    full_out = [torch.empty((s[1].shape[-2], N), device=dev) for s in stems]
    win_src = sources(crop_stems, wins, device=True)
    win_out = [torch.empty((s[1].shape[-2], CROP), device=dev) for s in crop_stems]
    for _ in range(3):
        R.render_device(full_src, full_out); R.render_device(win_src, win_out)
    torch.cuda.synchronize()
    for k, (a, n) in enumerate(wins):                  # bit identity, in this run
        assert torch.equal(win_out[k], full_out[k % len(stems)][:, a:a + n]), (title, k)
    f_ms, w_ms = median_ms([lambda: R.render_device(full_src, full_out), lambda: R.render_device(win_src, win_out)], reps)
    # host path
    hf_src, hw_src = sources(stems), sources(crop_stems, wins)
    hf_out = [np.empty((s[1].shape[-2], N), np.float32) for s in stems]
    hw_out = [np.empty((s[1].shape[-2], CROP), np.float32) for s in crop_stems]
    R.render_host(hf_src, hf_out); R.render_host(hw_src, hw_out)
    for k, (a, n) in enumerate(wins):
        assert np.array_equal(hw_out[k], hf_out[k % len(stems)][:, a:a + n]), (title, k)
    hf_ms, hw_ms = median_ms([lambda: R.render_host(hf_src, hf_out), lambda: R.render_host(hw_src, hw_out)], reps // 2)
    tf = np.sum([transforms(*s, None) for s in stems], axis=0)
    tw = np.sum([transforms(*s, w) for s, w in zip(crop_stems, wins)], axis=0)
    crop_s = len(wins) * CROP / SR
    print("%s" % title)
    print("  transforms (RIR pairs, dry pairs, inverse): full stems %s, %d windows %s" % (tuple(tf), len(wins), tuple(tw)))
    # per crop: one full stem rendered and cropped afterwards, against one window
    print("  device: full %8.3f ms (%d stems)   %d x 4 s windows %8.3f ms   per crop: %.4f vs %.4f ms (%.1fx)" %
          (f_ms, len(stems), len(wins), w_ms, f_ms / len(stems), w_ms / len(wins),
           (f_ms / len(stems)) / (w_ms / len(wins))))
    print("  host:   full %8.3f ms (%d stems)   %d x 4 s windows %8.3f ms   per crop: %.4f vs %.4f ms (%.1fx); "
          "%.0f crop audio-s/s" % (hf_ms, len(stems), len(wins), hw_ms, hf_ms / len(stems), hw_ms / len(wins),
                                   (hf_ms / len(stems)) / (hw_ms / len(wins)), crop_s / (hw_ms / 1e3)))


if __name__ == "__main__":
    R = render.Renderer(0)
    print("device:", card())
    rng = np.random.default_rng(7)
    np.random.seed(7)
    t0 = time.time()
    spk = scene(rng, 8, 0, 480000, 40, 6, 4096)
    case("configs[1] speakers: 8 x (P = 40, C = 6, L = 4096, 30 s); one 4 s window per speaker", spk, 1, rng)
    sc = scene(rng, 2, 2, 960000, 40, 2, 4096)
    case("60 s scene: 2 moving (P = 40) + 2 static, C = 2, L = 4096; one 4 s window per stem", sc, 1, rng)
    sc3 = scene(rng, 3, 0, 960000, 40, 2, 4096)
    case("batch of 32 crops x 3 stems (60 s, P = 40, C = 2) in one call", sc3, 32, rng, reps=10)
    print("window == slice of the full render, bit for bit, in every case (%.0f s)" % (time.time() - t0))
