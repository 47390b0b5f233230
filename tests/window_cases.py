"""Time windows (ss_source.win_start / win_len): the seeded cases, windows and the documented read set that the CPU and
GPU tests share, and the CPU helpers of windowed and pooled slots: tables, blockings and staged read sets."""
import ctypes

import numpy as np

from direct_path import CASES as DIRECT_CASES, make_case as make_direct_case
from oracle import sonicsim_oracle as so
from sonicsim_b200 import _lib

B = 4096
KSPEC = 4096

# name: (mode, P, C, L, N, taps); mode 0 static, 1 bounds, 2 (idx, w)
CASES = dict(DIRECT_CASES)
CASES.update({
    "bounds3": (1, 6, 3, 300, 21000, 40),      # C * K = 3: a position's rows start on an odd row
    "long1": (1, 4, 1, 9000, 20000, 800),      # K = 3, C * K = 3
    "long8": (1, 3, 2, 32768, 40000, 800),     # K = 8
    "zeroseg": (1, 7, 2, 4097, 20000, 40),     # zero-length segments; L = 4097: K = 2
    "edge4096": (1, 5, 2, 4096, 20000, 40),
    "gridchosen": (1, 40, 2, 4096, 20000, 40), # short segments: the host's cost rule picks the grid
})


def make_case(name):
    """(x, h (P, C, L), idx, w, bounds, taps) as direct_path.make_case."""
    if name in DIRECT_CASES:
        return make_direct_case(name)
    mode, P, C, L, N, taps = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x = so.synth_dry(rng, N)
    h = so.synth_rirs(rng, P, C, L)
    if name == "zeroseg":
        bounds = np.array([0, 3000, 3000, 3000, 9000, 15000, 20000], np.int32)
    else:
        np.random.seed(len(name))
        idx, _ = so.setup_dynamic_interp(so.synth_path(rng, P), N)
        bounds = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)
    idx = np.repeat(np.arange(P - 1), np.diff(bounds)).astype(np.int32)
    w = np.concatenate([np.linspace(0, 1, n, endpoint=False) for n in np.diff(bounds)]).astype(np.float32)
    return x, h, idx, w, bounds, taps


def full_blocks(N, bounds, aligned):
    """The full plan's blocks (start, len, p_lo, p_hi) as ss_debug_plan reports them."""
    if not aligned:
        return [(s, min(B, N - s), 0, 0) for s in range(0, N, B)]
    out = []
    for sg in range(len(bounds) - 1):
        b0, n = int(bounds[sg]), int(bounds[sg + 1] - bounds[sg])
        out += [(b0 + B * q, min(B, n - B * q), sg, sg + 1) for q in range((n + B - 1) // B)]
    return out


def windows(name, N, bounds, aligned, seed=0):
    """The windows of the test matrix: whole stem, first / last sample, inside one block, exactly one block, straddling
    a waypoint (moving) and a random one."""
    blocks = full_blocks(N, bounds, aligned)
    mid = blocks[len(blocks) // 2]
    ws = [(0, N), (0, 1), (N - 1, 1), (mid[0] + 7, max(1, min(100, mid[1] - 8))), (mid[0], mid[1])]
    if bounds is not None:
        b = int(bounds[2])
        if 0 < b - 50 and b + 50 <= N:
            ws.append((b - 50, 100))
    if name == "zeroseg":
        ws.append((2500, 1000))                    # spans the two empty segments at 3000
    rng = np.random.default_rng(seed + sum(map(ord, name)))
    a = int(rng.integers(0, N - 1))
    ws.append((a, int(rng.integers(1, N - a + 1))))
    return ws


def _seg(bounds, n):
    P = len(bounds)
    return min(int(np.searchsorted(bounds[1:], n, side="right")), P - 2)


def read_set(mode, P, C, L, N, bounds, aligned, win, normalize=False, host_visible=True):
    """The read set documented in include/sonicsim_b200.h: dry samples [xa, xb), idx / w entries [ia, ib), RIR positions
    [pa, pb]."""
    ws, wl = win
    K = (L + B - 1) // B
    blocks = full_blocks(N, bounds if mode == 1 else None, aligned)
    kept = [i for i, b in enumerate(blocks) if b[0] < ws + wl and b[0] + b[1] > ws]
    k0, k1 = kept[0], kept[-1] + 1
    g0 = max(0, k0 - (K - 1)) & ~1
    g1 = min(len(blocks), (k1 + 1) & ~1)
    xa, xb = max(0, blocks[g0][0] - B), min(N, blocks[g1 - 1][0] + B)
    ia, ib = blocks[k0][0], blocks[k1 - 1][0] + blocks[k1 - 1][1]
    if mode == 0:
        pa, pb = 0, 0
    elif normalize or mode == 2 or not host_visible:
        return (xa, xb), (ia, ib), (0, P - 1)
    elif aligned:
        pa, pb = blocks[k0][2], blocks[k1 - 1][3]
    else:
        pa, pb = _seg(bounds, ia), _seg(bounds, ib - 1) + 1
    ck = C * K
    r0, r1 = (pa * ck) & ~1, min(P * ck, ((pb + 1) * ck + 1) & ~1)
    return (xa, xb), (ia, ib), (r0 // ck, (r1 - 1) // ck)


def poison(x, h, idx, w, rs):
    """Copies of the inputs with everything outside the read set `rs` replaced: NaN for samples and taps, an
    out-of-range position for idx."""
    (xa, xb), (ia, ib), (pa, pb) = rs
    x2 = np.full_like(x, np.nan)
    x2[xa:xb] = x[xa:xb]
    h2 = np.full_like(h, np.nan)
    h2[pa:pb + 1] = h[pa:pb + 1]
    idx2 = w2 = None
    if idx is not None:
        idx2 = np.full_like(idx, 1 << 20)
        idx2[ia:ib] = idx[ia:ib]
        w2 = np.full_like(w, np.nan)
        w2[ia:ib] = w[ia:ib]
    return x2, h2, idx2, w2


def _p(a):
    return None if a is None else ctypes.c_void_p(a.ctypes.data)


def _k(L):
    return (L + B - 1) // B


def _needs_numpy(N, bounds, aligned, K, wl):
    """g1 - g0 of the table every start in [0, N - wl] needs, from the full plan (full_blocks)."""
    blk = np.array(full_blocks(N, bounds, aligned), np.int64)
    starts, ends = blk[:, 0], blk[:, 0] + blk[:, 1]
    ws = np.arange(N - wl + 1)
    k0 = np.searchsorted(ends, ws, side="right")
    k1 = np.searchsorted(starts, ws + wl, side="left")
    g0 = np.maximum(k0 - (K - 1), 0) & ~1
    g1 = np.minimum(len(blk), (k1 + 1) & ~1)
    return g1 - g0


def _random_bounds(rng, P, N, short):
    cuts = np.sort(rng.integers(0, (min(N, 3000) if short else N) + 1, P - 2))
    return np.ascontiguousarray(np.concatenate([[0], cuts, [N]]), np.int32)


def _choice(bounds, N, P, L):
    """The blocking the library picks for one candidate on its own (ss_debug_plan), 1 = aligned."""
    lib = _lib.load()
    item = _lib.SsSource(x=1, out=1, bounds=bounds.ctypes.data, bounds_host=bounds.ctypes.data, N=N, P=P, C=1, L=L,
                         mode=_lib.SS_MOVING_BOUNDS, rir=1)
    blk = np.zeros((N // B + P + 8, 4), np.int32)
    aligned = ctypes.c_int32()
    assert lib.ss_debug_plan(ctypes.byref(item), blk.ctypes.data, blk.shape[0], ctypes.byref(aligned)) > 0
    return aligned.value


class EmuCand:
    """One candidate: dry x, trajectory (None: static), RIRs and their emulated bank (with a direct set when taps > 0)."""

    def __init__(self, emu, rng, N, P, C, L, taps, short=False):
        self.N, self.P, self.C, self.L, self.K = N, P, C, L, _k(L)
        self.x = so.synth_dry(rng, N)
        self.bounds = None if P == 1 else _random_bounds(rng, P, N, short)
        h = so.synth_rirs(rng, P, C, L)
        sets = 2 if taps else 1
        self.spec = np.full((sets * P * C * self.K, KSPEC), np.nan, np.complex64)
        self.cut = np.zeros(P * C, np.int32) if taps else None
        emu.emu_bank_create(_p(h), P, C, L, 0, taps, _p(self.spec), _p(self.cut))
        self.direct = 1 if taps else 0

    def aligned_alone(self):
        return 0 if self.P == 1 else _choice(self.bounds, self.N, self.P, self.L)


def stage_cap(emu, cands, wl):
    N = np.array([c.N for c in cands], np.int32)
    P = np.array([c.P for c in cands], np.int32)
    K = np.array([c.K for c in cands], np.int32)
    out = np.zeros(2, np.int32)
    if cands[0].P == 1:
        emu.emu_stage_cap(None, None, _p(N), _p(P), _p(K), len(cands), cands[0].C, wl, _p(out))
    else:
        off = np.cumsum([0] + [c.P for c in cands[:-1]]).astype(np.int64)
        flat = np.ascontiguousarray(np.concatenate([c.bounds for c in cands]), np.int32)
        emu.emu_stage_cap(_p(flat), _p(off), _p(N), _p(P), _p(K), len(cands), cands[0].C, wl, _p(out))
    return int(out[0]), int(out[1])


def stage_set_np(N, P, C, K, bounds, ws, wl):
    """stage_set (ss_phases.cuh) in NumPy over an array of starts ws: (xa, xb, row0, rows) as int64 arrays.  The dry span
    [ws - (K + 2) 4096, ws + wl + 2 * 4096) clamped to [0, N); the rows of every position whose segment holds a sample of
    it and the one after, widened to row pairs and clipped to the bank (window_rows)."""
    ws = np.asarray(ws, np.int64)
    xa = np.maximum(ws - (K + 2) * B, 0)
    xb = np.minimum(ws + wl + 2 * B, N)
    if P > 1:
        inner = np.asarray(bounds, np.int64)[1:P]             # seg_of: bounds[1..P-1] <= n, clamped to P - 2
        pa = np.minimum(np.searchsorted(inner, xa, side="right"), P - 2)
        pb = np.minimum(np.searchsorted(inner, xb - 1, side="right"), P - 2) + 1
    else:
        pa, pb = np.zeros_like(ws), np.zeros_like(ws)
    ck = C * K
    r0 = (pa * ck) & ~1
    r1 = np.minimum(((pb + 1) * ck + 1) & ~1, P * ck)
    return xa, xb, r0, r1 - r0


def _bad_bounds(N=40960):
    """Bounds tables outside the contract (ascending from 0 to N): a huge interior waypoint that would make the aligned
    planner emit ~10^5 blocks, a descending step, a last entry != N, a first entry != 0."""
    good = np.array([0] + [2048 + 4096 * k for k in range(9)] + [38000, N], np.int64)
    huge = good.copy(); huge[-2] = 400000000
    desc = good.copy(); desc[3], desc[4] = desc[4], desc[3]
    short = good.copy(); short[-1] = N - 5
    late = good.copy(); late[0] = 100
    return good, [huge, desc, short, late]


def _host_aligned(mode, P, C, L, N, bounds):
    """The blocking the library picks with the trajectory on the host (ss_debug_plan)."""
    from sonicsim_b200 import render
    R = render.default_renderer()
    if mode != 1:
        return 0
    b = np.ascontiguousarray(bounds, np.int32)
    it = _lib.SsSource(x=1, rir=1, out=1, bounds=b.ctypes.data, N=N, P=P, C=C, L=L, mode=1, bounds_host=b.ctypes.data)
    cap = (N + 4095) // 4096 + P
    out = np.zeros((cap, 4), np.int32)
    al = ctypes.c_int32()
    assert R.lib.ss_debug_plan(ctypes.byref(it), out.ctypes.data, cap, ctypes.byref(al)) > 0
    return al.value
