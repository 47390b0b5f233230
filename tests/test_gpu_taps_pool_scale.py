"""Tap-form host pools (rir_bank(host=True, form="taps"), SS_BANK_TAPS) at training scale against float64.  A slot of a
tap-form pool stages its rows of taps (window_rows: whole positions, from an even row to past the last row's partner)
and one k_prepare launch turns them into the spectra its view names; everything after that - stage_set, stage_cap,
stage_head, take_view, k_blocks, the render kernels - is the code a spectral host pool's slot runs, so a fault there
gives the same wrong bits in both.  Every case here builds three arms from the same candidates - a device pool, a
spectral host pool and a tap-form host pool - and checks (i) that they give the same bits, starts, `used` and error
bits, and (ii) every stem of the tap arm sample by sample against float64 (render_reference.check_render through
ScaleCand.check on a thread pool; a normalised bank against the RIRs divided by their abs-max in float32, a pool with
loudness gains against the reference times its float32 gain, direct stems against direct_path_rirs).  Outputs lie in
NaN-filled buffers with sentinels on both sides (mix_reference.Out).
  A. staged crops of the grid, aligned (direct sets), mixed-K (C = 1, K = 1..4, and one moving candidate at L = 32768)
     and static (C = 5) pools, plain and normalised (abs-max 0.6: k_bank_taps divides every tap); the starts of
     test_gpu_host_pool_scale A, and windows whose first position p has odd p * C * K (row0 rounded down into position
     p - 1) or that end on the last row of an odd P * C * K (paired with make_row_h's absent row), both asserted to
     occur;
  B. training scale: configs[1] speakers with direct targets under the default and a small chunk budget, P = 60 speakers
     with random cuts and loudness gains, and a plan of 1056 tap slots of K = 1..3 whose launches are the spectral
     host-pool plan's plus one, as one graph;
  C. builds whose copy batches split stem groups (48 P = 60 speakers at K = 2) and a candidate whose tap copy alone
     exceeds 256 MiB: level tables, LUFS, loudness gains and pair gains equal the spectral twin's bit for bit, LUFS the
     float64 BS.1770 oracle and tables the long-double prefix.
No test holds more than 2 GB of pinned host memory in banks and pools (as counted by their host_nbytes)."""
import numpy as np
import pytest

from chunk_budget import DEFAULT_CHUNK_BYTES, chunk_budget  # noqa: F401  (fixture)
from draw_reference import TABLE_TOL, gappy_dry
from gpu_plumbing import _R
from oracle import sonicsim_oracle as so
from pool_worlds import (A_LENS, STEM_BYTES, Pools, Probes, ScaleCand, _hold, _random_cuts, _training, a_aligned,
                         a_grid, a_mixed_k, a_static, b_configs1, copy_batches, d_giant, d_speakers, host_alone,
                         probe_starts, read_set, report, stem_groups, table_error)
from render_reference import delay_rirs, graded_dry
from window_cases import _choice, stage_set_np

pytestmark = pytest.mark.gpu

RATE = 16000
B = 4096
SMALL_CHUNK = 2 << 20
FORMS = ("spectra", "taps")


def row_parity(c, ws, wl):
    """window_rows of the window's read set restated (stage_set_np's positions): (its first position p has odd
    p * C * K, so that row0 is rounded down to the last row of position p - 1; its rows end on the last row of an odd
    P * C * K, which pairs with make_row_h's absent row)."""
    xa, xb, r0, rows = (int(v[0]) for v in stage_set_np(c.N, c.P, c.C, c.K, c.b, [ws], wl))
    ck = c.C * c.K
    if c.P > 1:
        pa = min(int(np.searchsorted(np.asarray(c.b[1:c.P], np.int64), xa, side="right")), c.P - 2)
    else:
        pa = 0
    return (pa * ck) % 2 == 1, r0 + rows == c.P * ck and (c.P * ck) % 2 == 1


# ----------------------------------------------------------------------------------------- A. staged crops
def a_mixed_k_long(rng):
    """a_mixed_k (C = 1, K = 1..4) and a moving candidate at L = 32768 (K = 8)."""
    N, P = 100003, 5
    return a_mixed_k(rng) + [ScaleCand(graded_dry(rng, N), delay_rirs(rng, P, 1, 32768)[0],
                                       np.round(np.linspace(0, N, P)).astype(np.int32))]


# kind: (candidates, direct sets, render kernel, parities of window_rows that must occur)
A_POOLS = {"grid": (a_grid, False, "k_render<0,0>", {"row0"}),
           "aligned": (a_aligned, True, "k_render_fast", set()),
           "mixed-K": (a_mixed_k_long, False, "k_render<1,0>", {"row0", "end"}),
           "static": (a_static, False, "k_render_fast static", {"end"})}


@pytest.mark.parametrize("norm", ["plain", "normalised"])
@pytest.mark.parametrize("kind", list(A_POOLS))
def test_staged_tap_crops_at_every_read_set_edge(kind, norm):
    make, taps, variant, parities = A_POOLS[kind]
    R = _R()[1]
    rng = np.random.default_rng(2600 + len(kind))
    cands = make(rng)
    if norm == "normalised":                     # abs-max 0.6 (delay RIRs peak at exactly 1): every tap divided
        cands = [ScaleCand(c.x, c.h * np.float32(0.6) / np.float32(np.abs(c.h).max()), c.b) for c in cands]
        assert all(np.abs(c.h).max() not in (0.0, 1.0) for c in cands)
    pl = Pools(cands, taps=taps, form=FORMS, normalize=norm == "normalised")
    assert pl.arms == [False, True, "taps"] and pl.pools["taps"].resident == "host"
    assert pl.variant == variant, (kind, pl.variant)
    _hold(pl)
    k = 8
    n_min = min(c.N for c in cands)
    fixed = [n_min - wl for wl in A_LENS]
    pr = Probes(pl, A_LENS, k, fixed)
    sets = 2 if taps else 1
    key = "A %s %s" % (variant, norm)
    try:
        R.check_device_errors()
        queues = []
        for wl in A_LENS:                      # the largest read sets first, so that the full areas run side by side
            q = [read_set(c, s, wl, sets) + (i, s) for i, c in enumerate(cands) for s in probe_starts(c, wl, rng)]
            for i, c in enumerate(cands):      # and starts whose first position has odd p * C * K
                for s in rng.integers(0, c.N - wl + 1, 24):
                    if row_parity(c, int(s), wl)[0]:
                        q.append(read_set(c, int(s), wl, sets) + (i, int(s)))
                        break
            q.sort(key=lambda t: -t[0])
            queues.append(q)
        runs = max(-(-len(q) // k) for q in queues)
        seen = {"row0": 0, "end": 0}
        for r in range(runs):
            pk, st = [], []
            for wl, f, q in zip(A_LENS, fixed, queues):
                take = q[r * k:(r + 1) * k]
                while len(take) < k:                   # the rest: random picks and starts
                    i = int(rng.integers(0, len(cands)))
                    take.append((0, -1, -1, i, int(rng.integers(0, cands[i].N - wl + 1))))
                last = int(rng.integers(0, len(cands)))
                pk += [t[3] for t in take] + [last]
                st += [t[4] for t in take] + [0]
                for i, s in [(t[3], t[4]) for t in take] + [(last, f)]:
                    odd0, odd_end = row_parity(cands[i], s, wl)
                    seen["row0"] += odd0
                    seen["end"] += odd_end
            pr.run(pk, st)
            assert pr.launches["taps"] == pr.launches[True] + 1, pr.launches
            pr.check(key, "%s %s run %d" % (kind, norm, r))
        # the pairing cases of window_rows this pool can have, from the plan's own picks and starts
        assert {p for p, n in seen.items() if n} == parities, (kind, seen)
        R.check_device_errors()
        print("\n%s %s: %d runs of %d slots x 3 arms; windows with odd first-position rows %d, ending on an odd "
              "P * C * K %d" % (kind, norm, runs, len(pr.slots), seen["row0"], seen["end"]))
        report("A")
    finally:
        pr.close()
        pl.close()


# ----------------------------------------------------------------------------------------- B. training scale
@pytest.mark.parametrize("budget", ["default", "small"])
def test_training_configs1_tap_pool(budget, chunk_budget):
    R = chunk_budget(DEFAULT_CHUNK_BYTES if budget == "default" else SMALL_CHUNK)
    rng = np.random.default_rng(2701)
    spk, noi = b_configs1(rng)
    pools = {"spk": Pools(spk, taps=True, levels="mono", form=FORMS), "noi": Pools(noi, form=FORMS)}
    _hold(*pools.values())
    try:
        n = _training(pools, [("spk", True), ("spk", True), ("noi", False)], "configs1 taps %s" % budget)
        assert n["taps"] == n[True] + 1, n
        report("B configs1 taps %s" % budget)
    finally:
        for p in pools.values():
            p.close()
    assert R


def test_training_p60_tap_pool_with_gains():
    """P = 60 with random cuts (some candidates on the grid) over 24 shared RIR sets, loudness targets; 2 speakers, a
    noise and a music per example."""
    rng = np.random.default_rng(2702)
    N, P, C = 30 * RATE, 60, 6
    rirs = [so.synth_rirs(rng, P, C, 4096) for _ in range(24)]
    spk = [ScaleCand(gappy_dry(rng, N) if j % 3 == 0 else so.synth_dry(rng, N), rirs[j % 24],
                     _random_cuts(rng, P, N, None if j % 4 else 60000)) for j in range(32)]
    assert {_choice(c.b, N, P, 4096) for c in spk} == {0, 1}
    stat = [ScaleCand(so.synth_dry(rng, N - 1000 * j),
                      (rng.standard_normal((1, C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32), None)
            for j in range(12)]
    targets = [float(rng.uniform(-30, -16)) if j % 5 else None for j in range(len(spk))]
    pools = {"spk": Pools(spk, levels="mono", lufs=targets, share=[j % 24 for j in range(len(spk))], form=FORMS),
             "noi": Pools(stat[:6], form=FORMS), "mus": Pools(stat[6:], form=FORMS)}
    _hold(*pools.values())
    try:
        L = {a: pools["spk"].pools[a].loudness for a in pools["spk"].arms}
        for a in L:
            assert L[a].tobytes() == L["taps"].tobytes(), a
        assert not np.isnan(L["taps"][1]).any() and np.isnan(L["taps"][0]).all()
        n = _training(pools, [("spk", False), ("spk", False), ("noi", False), ("mus", False)], "P=60 taps gains")
        assert n["taps"] == n[True] + 1, n
        report("B P=60 taps gains")
    finally:
        for p in pools.values():
            p.close()


def test_many_tap_slots():
    """1056 slots of a tap-form pool of K = 1..3 and odd and even P * C * K, at two window lengths: one transform launch
    whose CTA prefix runs over every slot, with its own cap_rows per window length and its own rows per pick."""
    R = _R()[1]
    rng = np.random.default_rng(2703)
    cands = []
    for j in range(6):
        N, P, L = 20001 + 1001 * j, 3 + j % 3, (2000, 5000, 9000)[j % 3]
        cands.append(ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 1, L), _random_cuts(rng, P, N)))
    assert {(c.P * c.K) % 2 for c in cands} == {0, 1}
    pl = Pools(cands, form=FORMS)
    _hold(pl)
    lens, k = [1500, 3001], 527
    pr = Probes(pl, lens, k, [123, 77])
    n = len(pr.slots)
    assert n == 1056
    try:
        for run in range(2):
            pk = rng.integers(0, len(cands), n)
            st = [int(rng.integers(0, cands[p].N - wl + 1)) for p, (wl, _) in zip(pk, pr.slots)]
            pr.run(pk, st)
            pr.check("B many taps", "many taps run %d" % run)
        launches = pr.launches
        chunks = launches[False] / 3                     # k_blocks, k_prepare and the render per chunk
        print("\nmany tap slots: %d slots, %g chunks, launches per run %s (device, spectral host, tap host)" %
              (n, chunks, launches))
        assert launches["taps"] == launches[True] + 1 == launches[False] + 2 and chunks > 1, launches
        for p in pr.plans.values():
            assert p.is_graph()
        R.check_device_errors()
        report("B many taps")
    finally:
        pr.close()
        pl.close()


# ----------------------------------------------------------------------------------------- C. builds across batches
@pytest.mark.parametrize("kind", ["speakers", "giant"])
def test_tap_builds_across_copy_batches(kind):
    render, R = _R()
    rng = np.random.default_rng(2901 if kind == "speakers" else 2902)
    cands = d_speakers(rng, L=8192) if kind == "speakers" else d_giant(rng, P_giant=700)
    C = cands[0].C
    first, _ = stem_groups(C, [c.N for c in cands])
    batches, cap = copy_batches(C, cands, first, "taps")
    inside = [s for s in batches if s not in first]
    print("\n%s: stem groups %s, tap copy batches %s, copy buffer %d bytes" % (kind, first, batches, cap))
    if kind == "speakers":
        assert inside, (first, batches)                   # a tap batch boundary strictly inside a stem group
        unmeasured = {inside[0], first[1], first[1] - 1}
        silent = {inside[0] - 1}
    else:
        assert 4 * B * 700 * C * 3 > STEM_BYTES and cap > STEM_BYTES and 2 in batches and 3 in batches, (batches, cap)
        unmeasured, silent = {1}, {3}                      # on each side of the giant
    for j in silent:
        cands[j].x[:] = 0.0
    trng = np.random.default_rng(2903)
    targets = [None if j in unmeasured else float(trng.uniform(-30, -14)) for j in range(len(cands))]
    refs = [host_alone(R, render, c, t) for c, t in zip(cands, targets)]
    oracle = [None if t is None or j in silent else
              so.bs1770_integrated_loudness(host_alone(R, render, c, None)[0].T.astype(np.float64), RATE, 0.4,
                                            up_to_8_channels=True) for j, (c, t) in enumerate(zip(cands, targets))]
    n_max = max(c.N for c in cands)
    dry = [so.synth_dry(rng, n_max) * np.float32(0.7), gappy_dry(rng, n_max + 3)]
    pt = np.array([[float(trng.uniform(-28, -16)) for _ in cands] for _ in dry])
    pt[0, 0] = np.nan
    worst_tab = worst_db = 0.0
    for levels in ("mono", "channels"):
        twin = {}                                          # one form at a time: under 2 GB of pinned memory
        for form in FORMS:
            pl = Pools(cands, levels=levels, lufs=targets, host_only=True, form=form)
            dp = R.dry_pool(dry, host=True)
            _hold(pl)
            try:
                p = pl.pools[True if form == "spectra" else "taps"]
                assert p.resident == "host" and (pl.banks[0].form == form)
                pg = R.pair_gains(p, dp, pt, sr=RATE) if levels == "mono" else None
                twin[form] = (p.loudness, [p.level_table(i).cpu().numpy() for i in range(p.n)],
                              None if pg is None else pg.loudness)
                if pg is not None:
                    pg.close()
            finally:
                dp.close()
                pl.close()
        (Ls, Qs, Gs), (Lt, Qt, Gt) = twin["spectra"], twin["taps"]
        assert Ls.tobytes() == Lt.tobytes(), (kind, levels)
        if levels == "mono":                               # pair gains: every (dry signal, candidate) pair measured
            assert Gs.tobytes() == Gt.tobytes(), kind
            assert np.isnan(Gt[0, 0]).all() and not np.isnan(Gt[1]).any()
        for i, (c, t) in enumerate(zip(cands, targets)):
            what = (kind, levels, i)
            q = Qt[i]
            assert np.array_equal(q, Qs[i]), what
            y, lo = refs[i]
            if t is None:
                assert np.isnan(Lt[i]).all(), what
            else:
                assert (Lt[i, 0], Lt[i, 1]) == lo, (what, Lt[i], lo)
                if i in silent:
                    assert np.isneginf(Lt[i, 0]), what
                else:
                    d = abs(Lt[i, 0] - oracle[i])
                    assert d < 1e-6, (what, Lt[i, 0], oracle[i])
                    worst_db = max(worst_db, d)
            r = table_error(q, y, levels == "mono")
            assert r <= TABLE_TOL, (what, r / TABLE_TOL)
            worst_tab = max(worst_tab, r)
    print("%s: worst table error %.3g x TABLE_TOL, worst loudness vs the oracle %.3g dB" %
          (kind, worst_tab / TABLE_TOL, worst_db))
