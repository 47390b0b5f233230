"""Time windows (ss_source.win_start / win_len): the seeded cases, windows and the documented read set that the CPU and
GPU tests share."""
import numpy as np

from direct_path import CASES as DIRECT_CASES, make_case as make_direct_case
from oracle import sonicsim_oracle as so

B = 4096

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
