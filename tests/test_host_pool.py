"""Host pools on the CPU, through the kernels' own helpers (exported by tests/emu/ss_emu_stage.cu): the read set k_stage
copies for a pooled slot of a host pool (stage_set) and the staging area a plan sizes for it (stage_cap).
  - the staged set holds every dry sample and RIR row the windowed render reads - the dry windows of the table's blocks
    (window_blocks) and window_rows of the positions of the blocks that meet the window;
  - it never exceeds the slot's staging area, which is the largest set of any candidate at any start;
  - the head of k_blocks over the staged view (take_view) builds the same Source, block table, work items, h_row0 / h_rows
    origin and direct-set rows as over the full candidate (pick_slot), and the slot renders the same bits from copies
    that hold the read set and NaN everywhere else;
  - a NumPy restatement of stage_set matches the kernels' at sampled starts, and over every start of training-shaped
    candidates (N = 480 000, P in {40, 60} with runs of short segments, K = 1..4, static and moving) stage_cap equals
    the largest read set exactly."""
import numpy as np
import pytest

from emu import build_emu
from window_cases import B, EmuCand, _k, _p, stage_cap, stage_set_np


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_stage")


def _slot(emu, c, aligned, k_pool, ws, wl, render):
    outs = [np.full((c.C, wl), np.nan, np.float32) for _ in range(4)]
    info = np.zeros(15, np.int32)
    emu.emu_stage_slot(_p(c.x), _p(c.spec), _p(c.cut), _p(c.bounds), c.N, c.P, c.C, c.L, 0 if c.P == 1 else 1,
                       aligned, k_pool, ws, wl, c.direct, int(render), *[_p(o) for o in outs], _p(info))
    return info, outs


def _check_tables(info, c, ws, wl):
    xa, xb, row0, rows = (int(v) for v in info[:4])
    # the staged set holds the read set
    assert xa <= info[4] and info[5] <= xb, (ws, wl, info[:8].tolist())
    assert row0 <= info[6] and info[6] + info[7] <= row0 + rows, (ws, wl, info[:8].tolist())
    assert row0 % 2 == 0 and 0 <= row0 and row0 + rows <= c.P * c.C * c.K
    # the staged view builds the same Source, table and items; the full run's rows start at 0, the staged at row0
    assert info[8] == 1, (ws, wl)
    assert info[9:13].tolist() == [0, c.P * c.C * c.K, row0, rows], (ws, wl, info[9:13].tolist())
    assert info[13:15].tolist() == ([c.P * c.C * c.K, rows] if c.direct else [-1, -1])
    return xb - xa, rows


def _starts(c, wl, every):
    last = c.N - wl
    if every:
        return list(range(last + 1))
    s = {0, last, last // 2, min(last, (c.K + 2) * B)}
    for b in ([] if c.bounds is None else c.bounds[1:-1]):      # segment edges, on both sides
        for d in (-1, 0, 1):
            if 0 <= b + d <= last:
                s.add(int(b + d))
    for q in range(0, c.N, B):                                  # grid block edges
        for d in (-1, 0):
            if 0 <= q + d <= last:
                s.add(q + d)
    return sorted(s)


CASES = [  # (P, C, L list, taps, N range, wl, every start)
    (1, 3, [1000], 0, (9000, 13000), 3000, True),
    (1, 2, [9000, 16384], 40, (20000, 30000), 6000, False),
    (4, 2, [4096], 0, (9000, 12000), 2500, True),
    (5, 3, [3000], 40, (20000, 40000), 7000, False),
    (3, 1, [4097, 9000, 16000], 0, (20000, 40000), 9000, False),
    (6, 2, [2000, 8192, 12289], 40, (25000, 40000), 5000, False),
]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_staged_set_holds_the_read_set_within_capacity(emu, case):
    """Aligned and grid blocking, K = 1..4, static and moving, with and without a direct set: at every start of the small
    cases and at the first, last, segment- and block-edge starts of the larger ones, the staged set holds what the slot
    reads, and the slot's staging area (stage_cap over the pool) holds the staged set; the capacity is reached."""
    P, C, Ls, taps, (n_lo, n_hi), wl, every = CASES[case]
    rng = np.random.default_rng(100 + case)
    cands = [EmuCand(emu, rng, int(rng.integers(n_lo, n_hi)), P, C, L, taps, short=i % 2 == 1)
             for i, L in enumerate(Ls * 2)]
    k_pool = max(c.K for c in cands)
    aligned = int(all(c.aligned_alone() for c in cands)) if P > 1 else 0
    cap_rows, cap_x = stage_cap(emu, cands, wl)
    most_rows, most_x = 0, 0
    for c in cands:
        for ws in _starts(c, wl, every):
            info, _ = _slot(emu, c, aligned, k_pool, ws, wl, render=False)
            nx, rows = _check_tables(info, c, ws, wl)
            assert rows <= cap_rows and nx + 8 <= cap_x, (ws, rows, cap_rows, nx, cap_x)
            most_rows, most_x = max(most_rows, rows), max(most_x, nx + 8)
    if every:                                                   # every start was tried: the capacity is exact
        assert (most_rows, most_x) == (cap_rows, cap_x)


def test_both_blockings_and_every_k_are_covered():
    seen = set()
    rng_cases = [(P, Ls) for P, C, Ls, *_ in CASES]
    for P, Ls in rng_cases:
        for L in Ls:
            seen.add(("static" if P == 1 else "moving", _k(L)))
    assert {k for _, k in seen} == {1, 2, 3, 4} and {"static", "moving"} <= {m for m, _ in seen}


def _emu_stage_set(emu, c, ws, wl):
    out = np.zeros(4, np.int32)
    emu.emu_stage_set(c.N, c.P, c.C, c.K, _p(c.bounds), int(ws), wl, _p(out))
    return out.tolist()


class Shape:
    """A candidate's shape alone (no signals): N, P, C, K and its trajectory."""

    def __init__(self, N, P, C, K, bounds):
        self.N, self.P, self.C, self.K, self.bounds = N, P, C, K, bounds


def training_bounds(rng, P, N):
    """Random cuts over [0, N) with a run of segments shorter than 4096 (some empty) somewhere inside."""
    k = P // 3
    at = int(rng.integers(0, N - 12000))
    short = at + np.sort(rng.integers(0, 12000, k))
    cuts = np.sort(np.concatenate([short, rng.integers(0, N + 1, P - 2 - k)]))
    return np.ascontiguousarray(np.concatenate([[0], cuts, [N]]), np.int32)


TRAIN_N = 480000
TRAIN_LENS = [64000, 3 * B + 5, 1000]


def training_shapes(seed):
    """Static and moving (P = 40, 60) training-shaped candidates with K = 1..4 and C in {6, 1, 3}."""
    rng = np.random.default_rng(seed)
    out = []
    for K in (1, 2, 3, 4):
        for P, C in ((1, 6), (40, 6), (60, 6), (40, 1), (60, 3)):
            out.append(Shape(TRAIN_N, P, C, K, None if P == 1 else training_bounds(rng, P, TRAIN_N)))
    return out


def test_numpy_stage_set_matches_the_kernels(emu):
    """The NumPy restatement against emu_stage_set (the kernels' own stage_set) at every segment edge +-1, the
    maximisers of stage_cap, both clamps and random starts of the training shapes and of short candidates."""
    lib = emu
    rng = np.random.default_rng(31)
    shapes = training_shapes(30) + [Shape(n, P, C, K, None if P == 1 else training_bounds(rng, P, n))
                                    for n, P, C, K in ((13001, 4, 2, 1), (20003, 6, 3, 3), (9002, 1, 5, 4))]
    n = 0
    for c in shapes:
        for wl in TRAIN_LENS:
            last = c.N - wl
            if last < 0:
                continue
            ws = {0, last, min(last, (c.K + 2) * B), min(last, (c.K + 2) * B - 1)}
            ws |= {int(v) for v in rng.integers(0, last + 1, 60)}
            for b in ([] if c.bounds is None else c.bounds[1:-1]):
                for d in (-1, 0, 1):
                    for v in (b + d, b + d + (c.K + 2) * B, b + d - wl - 2 * B):
                        if 0 <= v <= last:
                            ws.add(int(v))
            ws = np.array(sorted(ws), np.int64)
            got = np.stack(stage_set_np(c.N, c.P, c.C, c.K, c.bounds, ws, wl), axis=1)
            for w, g in zip(ws, got):
                assert g.tolist() == _emu_stage_set(lib, c, w, wl), (c.P, c.C, c.K, wl, int(w))
            n += len(ws)
    assert n > 10000


@pytest.mark.parametrize("wl", TRAIN_LENS)
def test_stage_cap_is_the_maximum_over_every_start(emu, wl):
    """N = 480 000, P in {40, 60} with random cuts that include segments shorter than 4096, K = 1..4, static and moving:
    stage_cap of each candidate alone, and of all the moving (and all the static) candidates of one C as one pool,
    equals the largest read set over every start in [0, N - len] exactly - rows, and dry samples + 8."""
    lib = emu
    shapes = training_shapes(40 + wl % 97)
    ws = np.arange(TRAIN_N - wl + 1, dtype=np.int64)
    most = []
    for c in shapes:
        xa, xb, _, rows = stage_set_np(c.N, c.P, c.C, c.K, c.bounds, ws, wl)
        m = (int(rows.max()), int((xb - xa).max()) + 8)
        assert stage_cap(lib, [c], wl) == m, (c.P, c.C, c.K, wl, stage_cap(lib, [c], wl), m)
        most.append(m)
    for static in (True, False):
        for C in {c.C for c in shapes}:
            group = [i for i, c in enumerate(shapes) if c.C == C and (c.P == 1) == static]
            if not group:
                continue
            want = (max(most[i][0] for i in group), max(most[i][1] for i in group))
            assert stage_cap(lib, [shapes[i] for i in group], wl) == want, (static, C, wl)


@pytest.mark.parametrize("case", range(len(CASES)))
def test_staged_slot_renders_the_same_bits(emu, case):
    """The slot rendered from copies of the read set (NaN everywhere else) against the slot over the full candidate:
    the same bits for the reverberant and the direct stem, at the first, last and edge starts and a few others."""
    P, C, Ls, taps, (n_lo, n_hi), wl, _ = CASES[case]
    rng = np.random.default_rng(200 + case)
    cands = [EmuCand(emu, rng, int(rng.integers(n_lo, n_hi)), P, C, L, taps, short=i % 2 == 1) for i, L in enumerate(Ls)]
    k_pool = max(c.K for c in cands)
    aligned = int(all(c.aligned_alone() for c in cands)) if P > 1 else 0
    for c in cands:
        starts = _starts(c, wl, False)
        pick = sorted({starts[0], starts[-1]} | set(rng.choice(starts, size=min(4, len(starts)), replace=False).tolist()))
        for ws in pick:
            info, (yf, ys, df, ds) = _slot(emu, c, aligned, k_pool, int(ws), wl, render=True)
            _check_tables(info, c, ws, wl)
            assert not np.isnan(yf).any() and np.array_equal(yf, ys), (case, ws)
            if taps:
                assert not np.isnan(df).any() and np.array_equal(df, ds), (case, ws)
