"""Host dry pools on the CPU, through the kernels' own helpers (exported by tests/emu/ss_emu_dry_stage.cu): a dry-picked
slot of a device pool whose dry samples k_stage stages from a host dry pool's arena.
  - the head of k_stage (stage_head) and the head of k_blocks over its view (take_view) build the same Source, block
    table, work items and h_row0 / h_rows origin as pick_pooled with a dry pick from a device dry pool, keep the bank's
    spectra, and report the same error bits for an out-of-range dry pick;
  - the slot renders the same bits from a staging copy holding only the whole float4s [xa & ~3, (xb + 3) & ~3) of the
    picked signal, NaN everywhere else, as from the whole signal: signals exactly N long with N % 4 != 0 and longer ones
    (with NaN past N), moving (K = 1..4, aligned and grid blocking) and static candidates, with and without a direct set,
    starts at 0, at N - len and at segment and block edges;
  - the staged span holds every dry sample the render reads, stays inside the arena's padded signal, and fits the dry
    count of stage_cap over the pool - the slot's staging area."""

import numpy as np
import pytest

from emu import build_emu
from window_cases import B, EmuCand, _p, stage_cap


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_dry_stage")


def _dry_slot(emu, c, d, aligned, k_pool, ws, wl, render, n_dry=1, dv=0):
    outs = [np.full((c.C, wl), np.nan, np.float32) for _ in range(4)]
    info = np.zeros(16, np.int32)
    emu.emu_dry_stage_slot(_p(c.x), _p(c.spec), _p(c.cut), _p(c.bounds), c.N, c.P, c.C, c.L, 0 if c.P == 1 else 1,
                           aligned, k_pool, ws, wl, c.direct, _p(d), d.size, n_dry, dv, int(render),
                           *[_p(o) for o in outs], _p(info))
    return info, outs


def _signals(rng, c):
    """The picked signals of a candidate: exactly N long, and longer with NaN past N (nothing past N may be read)."""
    exact = (rng.standard_normal(c.N) * 0.1).astype(np.float32)
    longer = np.full(c.N + 1 + int(rng.integers(0, 9000)), np.nan, np.float32)
    longer[:c.N] = (rng.standard_normal(c.N) * 0.1).astype(np.float32)
    return [exact, longer]


def _starts(c, wl):
    last = c.N - wl
    s = {0, last, min(last, (c.K + 2) * B)}
    for b in ([] if c.bounds is None else c.bounds[1:-1]):      # segment edges, on both sides
        for d in (-1, 0):
            if 0 <= b + d <= last:
                s.add(int(b + d))
    for q in range(B, c.N, 3 * B):                              # grid block edges
        for d in (-1, 0):
            if 0 <= q + d <= last:
                s.add(q + d)
    return sorted(s)


def _check(info, c, d, cap_x):
    x0, x1, xa, xb = (int(v) for v in info[:4])
    assert x0 == xa & ~3 and x1 == (xb + 3) & ~3 and 0 <= xa <= xb <= c.N
    assert x0 <= info[4] and info[5] <= x1, info[:6].tolist()          # the staged span holds the read set
    assert x1 <= (d.size + 3) & ~3                                       # inside the arena's padded signal
    assert x1 - x0 <= cap_x, (x1 - x0, cap_x)                            # and the slot's staging area
    assert info[6] == 1 and info[15] == 1
    rows = c.P * c.C * c.K
    assert info[7:11].tolist() == [0, rows, 0, rows]                     # a device pool's origin: the bank's rows
    assert info[11:13].tolist() == ([rows, rows] if c.direct else [-1, -1])
    assert info[13:15].tolist() == [0, 0]


CASES = [  # (P, C, L list, taps, N range, wl)
    (1, 3, [1000], 0, (9000, 13000), 3001),
    (1, 2, [9000], 40, (20000, 30000), 3 * B + 5),
    (4, 2, [4096], 40, (20000, 26000), 3001),
    (5, 3, [3000], 0, (20000, 40000), 3 * B + 5),
    (3, 1, [4097, 9000, 16000], 0, (30000, 40000), 3001),
    (6, 2, [2000, 8192, 12289], 40, (25000, 40000), 3 * B + 5),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_dry_only_staged_slot_matches_the_device_dry_pick(emu, case):
    """Tables, items and origins at every sampled start; bits of the render at 0, N - len and two edge starts, for a
    signal exactly N long (N % 4 != 0) and a longer one."""
    P, C, Ls, taps, (n_lo, n_hi), wl = CASES[case]
    rng = np.random.default_rng(300 + case)
    cands = []
    for i, L in enumerate(Ls):
        N = int(rng.integers(n_lo, n_hi))
        N += N % 4 == 0                                                 # N % 4 != 0
        cands.append(EmuCand(emu, rng, N, P, C, L, taps, short=i % 2 == 1))
    assert all(c.N % 4 for c in cands)
    k_pool = max(c.K for c in cands)
    aligned = int(all(c.aligned_alone() for c in cands)) if P > 1 else 0
    _, cap_x = stage_cap(emu, cands, wl)
    rendered = 0
    for c in cands:
        starts = _starts(c, wl)
        picks = {starts[0], starts[-1], starts[len(starts) // 2], starts[len(starts) // 3]}
        for d in _signals(rng, c):
            for ws in starts:
                info, outs = _dry_slot(emu, c, d, aligned, k_pool, ws, wl, ws in picks)
                _check(info, c, d, cap_x)
                if ws not in picks:
                    continue
                rendered += 1
                for dev, staged in ((outs[0], outs[1]), (outs[2], outs[3])) if c.direct else ((outs[0], outs[1]),):
                    assert np.isfinite(dev).all(), ws
                    assert np.array_equal(dev.view(np.uint32), staged.view(np.uint32)), ws
    assert rendered >= 6 * len(cands)


def test_out_of_range_dry_pick_is_clamped_as_k_blocks_clamps_it(emu):
    """A dry pick outside [0, n_dry) sets bit 16 in k_stage's head as in pick_pooled, and both take the same signal."""
    rng = np.random.default_rng(7)
    c = EmuCand(emu, rng, 21001, 4, 2, 4096, 0)
    d = (rng.standard_normal(c.N + 3) * 0.1).astype(np.float32)
    for dv in (-1, 2, 1 << 30):
        info, outs = _dry_slot(emu, c, d, 0, 1, 5000, 3001, True, n_dry=2, dv=dv)
        assert info[13:15].tolist() == [16, 16] and info[6] == 1
        assert np.array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
