"""Dry pools (ss_dry_pool_create, ss_plan_create_dry, render.DryPick) at training scale against float64.  A dry pick
changes only the slot's x at the head of k_blocks (pick_pooled -> pick_dry) and a table pointer in k_draw
(speaker_table), so a wrong pointer, slot mapping or offset gives finite, well-formed, wrong audio.  Every dry-picked
stem here is checked (i) bit for bit against render_device of the picked candidate with dry = signal[:N] at the same
window, and (ii) sample by sample against float64 (render_reference.check_render of render_f64(signal[:N], ...); a quiet
crop takes the scale-relative global rule of test_gpu_host_pool_scale, at 2^-5; direct stems against direct_path_rirs).  Outputs
lie in NaN-filled buffers with sentinels on both sides (test_gpu_plan_scale.Out); dry signals carry NaN tails that no
slot may read.  The float64 references run window by window (L - 1 samples of context) on a thread pool.
  A. one pool per kernel variant (grid, aligned with direct targets, K = 1..4, L = 32768, static L <= 4096 and
     L > 4096) over a dry pool of white, graded and impulse signals of different lengths; starts 0 and N - len of the
     picked candidate, ws % 4 in {1, 2, 3}, just past waypoints, clamped; windows 3001, 3 * 4096 + 5 and 64 000 (4 s);
     runs written on the device with no host synchronisation; the raw error bits of clamped picks, dry picks and starts;
  B. signal addressing: rows of an (n, T) tensor with odd T (every residue mod 16), slices at storage offsets 1 to 3, one
     far longer signal, rendered through aligned and grid slots, and their level tables;
  C. a plan of 1040 slots over two dry pools (dry-picked and plain slots of three pools, unpooled banked sources, a
     static source) under the default chunk budget and a small one; a second plan over the same dry pool in turn;
  D. k_draw's warp edges with dry-picked speakers (dry beacons: every try at least 29 dB from the threshold), and a
     training plan of 64 examples x (2 dry-picked speakers + a dry-picked noise) with mixtures;
  E. dry level tables at k_levels tile edges and unaligned signals, and a pool of 65 542 signals (two k_levels launches);
  F. lifetimes: a dry pool closed under two live plans, its caller's tensors dropped, and its memory returned."""
import gc

import numpy as np
import pytest
import torch

import draw_reference as dr
from chunk_budget import DEFAULT_CHUNK_BYTES, chunk_budget  # noqa: F401  (fixture)
from direct_path import direct_path_rirs
from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, dry_signal, render_check_inputs, rir_set
from draw_reference import NEAR_DB, TABLE_TOL, gappy_dry
from gpu_plumbing import _R, _device_errors, _rms, pmap, to
from mix_reference import Out, check_mixture, fold
from pool_worlds import (LARGE, NL, NN, NS, SMALL, DevPool, DryDrawPlan, ScaleCand, _bounds_of, _random_cuts,
                         a_aligned, a_mixed_k, a_static, d_cases, d_combos, dry_beacon, traj_beacon)
from window_cases import _choice

pytestmark = pytest.mark.gpu

RATE = 16000
B = 4096
TAPS = 40
NAN = float("nan")
STATS = {}                       # section / variant -> [worst local ratio, worst global relative RMS]
QUIET = {}                       # section / variant -> number of quiet crops held to the scale-relative rule


def _report(section):
    print()
    for k in sorted(STATS):
        if k.startswith(section):
            print("%-34s worst per-sample ratio %.3g (bound %.3g), worst global relative RMS %.3g (bound %.3g); "
                  "%d quiet crops" % (k, STATS[k][0], TAU_LOCAL, STATS[k][1], TAU_GLOBAL, QUIET.get(k, 0)))


# ------------------------------------------------------------------------------------------------ float64 checks
def f64_job(job):
    """One stem against float64: (key, worst local ratio, global relative RMS, quiet).  A crop of at least one block is
    held to the global bound, relative to its own RMS or, for a quiet crop (RMS under 2^-5 of its rounding scale's),
    relative to the scale's RMS.  Such a crop carries the rounding of its loud neighbours' transforms, which its own
    RMS does not measure: e.g. the K = 1 candidate of the mixed-K pool over a graded signal at 57708 + 12293 samples,
    two silent blocks and a quiet one behind a block 500 times louder, RMS 2^-5.7 of its scale's, error 3.1e-6 of its
    RMS and 6.1e-8 of the scale's."""
    key, label, x, c, a, wl, y, direct = job
    h = direct_path_rirs(c.h, TAPS) if direct else c.h
    y64, scale = render_check_inputs(x, h if c.P > 1 else h[0], c.mode, bounds=c.b, window=(a, wl))
    quiet = wl >= B and _rms(y64) < _rms(scale) / 32
    worst, g = check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL if wl >= B and not quiet else np.inf, n0=a,
                            label=label)
    if quiet:
        g = _rms(np.asarray(y, np.float64) - y64) / _rms(scale)
        assert g <= TAU_GLOBAL, "%s: quiet crop, global RMS %.3g of the scale's > %.3g" % (label, g, TAU_GLOBAL)
    return key, worst, g if wl >= B else 0.0, quiet


def check_f64(jobs):
    for key, worst, g, quiet in pmap(f64_job, jobs):
        s = STATS.setdefault(key, [0.0, 0.0])
        s[0], s[1] = max(s[0], worst), max(s[1], g)
        QUIET[key] = QUIET.get(key, 0) + int(quiet)


def check_stem(pl, i, xd, xh, s, wl, y, yd, key, label, jobs):
    """A dry-picked stem (and direct stem) of candidate i with dry signal xd (device) / xh (host) at start s: bits
    against render_device now, float64 queued in `jobs`."""
    c = pl.cands[i]
    if pl.bits[i]:
        ref, dref = pl.ref(i, xd, s, wl)
        assert np.array_equal(y, ref), (label, "bits")
    x = c.x if xh is None else xh[:c.N]
    jobs.append((key, label, x, c, s, wl, y, False))
    if pl.taps:
        assert not pl.bits[i] or np.array_equal(yd, dref), (label, "direct bits")
        jobs.append((key, label + " direct", x, c, s, wl, yd, True))


class DrySlots:
    """Dry-picked slots of one pool: `k` per window length, each with its own pick, dry pick and start in device
    memory, NaN-filled guarded outputs (and direct outputs)."""

    def __init__(self, pl, dp, lens, k):
        render, R = _R()
        self.pl, self.dp = pl, dp
        self.slots = [wl for wl in lens for _ in range(k)]
        n = len(self.slots)
        self.vals = torch.zeros((3, n), dtype=torch.int32, device="cuda")        # picks, dry picks, starts
        C = pl.cands[0].C
        self.outs = [Out(C, wl) for wl in self.slots]
        self.douts = [Out(C, wl) for wl in self.slots] if pl.taps else []
        srcs = [render.Pooled(pl.pool, self.vals[0, j], (self.vals[2, j], wl), pl.taps,
                              render.DryPick(dp, self.vals[1, j])) for j, wl in enumerate(self.slots)]
        self.plan = R.plan_device(srcs, [o.view() for o in self.outs],
                                  direct_outs=[o.view() for o in self.douts] if pl.taps else None)

    def run(self, vals):
        """One run with (3, n) device values and no host synchronisation; returns snapshots of every buffer."""
        for o in self.outs + self.douts:
            o.reset()
        self.vals.copy_(vals)
        self.plan.run()
        return [o.buf.clone() for o in self.outs + self.douts]

    def check(self, vals, snap, sig_d, sig_h, key, label, jobs):
        """Every slot of one run against the clamped pick, dry pick and start it must have rendered."""
        n = len(self.slots)
        for j, wl in enumerate(self.slots):
            i = min(max(int(vals[0][j]), 0), len(self.pl.cands) - 1)
            d = min(max(int(vals[1][j]), 0), len(sig_d) - 1)
            s = min(max(int(vals[2][j]), 0), self.pl.cands[i].N - wl)
            y = self.outs[j].get(snap[j])
            yd = self.douts[j].get(snap[n + j]) if self.pl.taps else None
            check_stem(self.pl, i, sig_d[d], sig_h[d], s, wl, y, yd, key,
                       "%s slot %d cand %d dry %d start %d len %d" % (label, j, i, d, s, wl), jobs)

    def close(self):
        self.plan.close()


# ----------------------------------------------------------------------------------------- A. kernel variants
A_LENS = [3001, 3 * B + 5, 64000]          # 64 000 samples: 4 s at 16 kHz
KINDS = ("white", "graded", "impulse")
TAILS = (0, 1, 2, 3, 5000, 77)             # NaN samples behind each signal's first n_max


def a_grid(rng):
    """Moving candidates with 59 segments of 0.3 to 3.8 k samples: grid blocking (generic k_render)."""
    out = []
    for j, N in enumerate((70001, 83002, 76003)):
        P = 60
        np.random.seed(510 + j)
        b = _bounds_of(so.setup_dynamic_interp(so.synth_path(rng, P), N)[0], P)
        assert _choice(b, N, P, B) == 0
        out.append(ScaleCand(so.synth_dry(rng, N), rir_set("delay" if j % 2 else "synth", rng, P, 3, B), b))
    return out


def a_long(rng):
    """Long RIRs (L = 32768: K = 8, and K = 5) at reduced N."""
    return [ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, L), np.round(np.linspace(0, N, P)).astype(np.int32))
            for N, P, L in ((90001, 5, 32768), (100002, 4, 20000), (80003, 6, 32768))]


def a_static_long(rng):
    return [ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, L), None)
            for N, L in ((66001, 8192), (70002, 12000), (80003, 5000))]


A_POOLS = {"grid": (a_grid, 0, "k_render<0,0>"), "aligned": (a_aligned, TAPS, "k_render_fast"),
           "mixed-K": (a_mixed_k, 0, "k_render<1,0> K=1..4"), "long": (a_long, 0, "k_render<1,0> L=32768"),
           "static": (a_static, 0, "k_render_fast static"), "static-long": (a_static_long, 0, "k_render<1,0> static")}


def dry_set(rng, n_max, n=6, tails=TAILS):
    """n dry signals, white, graded and impulse in turn, finite on [0, n_max) and NaN behind (the first exactly n_max
    long): host arrays and device tensors."""
    hs = []
    for j in range(n):
        x = np.full(n_max + tails[j % len(tails)], np.nan, np.float32)
        x[:n_max] = dry_signal(KINDS[j % 3], rng, n_max)
        if KINDS[j % 3] == "impulse":
            x[:n_max] = np.roll(x[:n_max], 5 * j)             # impulse trains at different phases
        hs.append(x)
    return hs, [to(x) for x in hs]


def a_starts(c, wl, rng):
    """0 and N - len, starts with ws % 4 in {1, 2, 3}, starts at and just past waypoints (block starts for a static
    candidate), all inside [0, N - len]; then two clamped starts, one past N - len and one below 0."""
    last = c.N - wl
    s = {0, last, max(0, last - 1)}
    for m in (1, 2, 3):
        v = int(rng.integers(0, last + 1))
        s.add(v - v % 4 + m)
    way = c.b[1:-1] if c.b is not None else np.arange(B, c.N, B)
    for q in way[::max(1, len(way) // 3)][:3]:
        s |= {int(q) + 1, int(q) + 2}
    return sorted(v for v in s if 0 <= v <= last) + [last + 1 + int(rng.integers(0, 50)), -1 - int(rng.integers(0, 3))]


@pytest.mark.parametrize("kind", list(A_POOLS))
def test_every_variant_and_window_edge(kind):
    make, taps, variant = A_POOLS[kind]
    render, R = _R()
    rng = np.random.default_rng(1100 + len(kind))
    cands = make(rng)
    assert 3 <= len(cands) <= 8
    pl = DevPool(cands, taps=taps)
    sig_h, sig_d = dry_set(rng, pl.n_max)
    dp = R.dry_pool(sig_d)
    assert dp.n_min == pl.n_max and dp.n == 6
    k = 8
    sl = DrySlots(pl, dp, A_LENS, k)
    key = "A %s" % variant
    try:
        R.check_device_errors()
        queues = []
        for wl in A_LENS:
            q = [(i, s) for i, c in enumerate(cands) for s in a_starts(c, wl, rng)]
            queues.append([(i, (n + wl) % dp.n, s) for n, (i, s) in enumerate(q)])    # every dry signal in turn
        runs = max(-(-len(q) // k) for q in queues)
        allv = np.zeros((runs, 3, len(sl.slots)), np.int32)
        for r in range(runs):
            for w, q in enumerate(queues):
                for j in range(k):
                    t = q[r * k + j] if r * k + j < len(q) else (int(rng.integers(0, len(cands))),
                                                                 int(rng.integers(0, dp.n)), 0)
                    allv[r, :, w * k + j] = t[0], t[1], t[2]
        dv = to(allv)
        snaps = [sl.run(dv[r]) for r in range(runs)]          # no host synchronisation between the runs
        assert sl.plan.is_graph()
        assert _device_errors(R) == 4                         # the clamped starts, of dry-picked slots
        jobs = []
        for r in range(runs):
            sl.check(allv[r], snaps[r], sig_d, sig_h, key, "%s run %d" % (kind, r), jobs)
        # one run with a clamped trajectory pick, a clamped dry pick and a clamped start in three different slots
        bad = allv[0].copy()
        bad[0, 0] = len(cands) + 3
        bad[1, 1] = -2
        bad[2, 2] = cands[bad[0, 2]].N - A_LENS[0] + 9
        snap = sl.run(to(bad))
        assert _device_errors(R) == 4 | 8 | 16
        sl.check(bad, snap, sig_d, sig_h, key, "%s clamped" % kind, jobs)
        sl.run(to(bad))
        with pytest.raises(IndexError):
            R.check_device_errors()
        R.check_device_errors()                               # cleared
        check_f64(jobs)
        print("\n%s: %d runs of %d dry-picked slots, %d stems against float64" % (kind, runs, len(sl.slots), len(jobs)))
        _report(key)
    finally:
        sl.close()
        dp.close()
        pl.close()


# ----------------------------------------------------------------------------------------- B. signal addressing
def table_check(q, x):
    """A device level table against the long-double prefix of signal x, within TABLE_TOL * Q[N]."""
    ref = dr.level_table(np.asarray(x, np.float32)[None], True, np.longdouble)
    assert q.shape == ref.shape and q[0] == 0.0
    err = float(np.max(np.abs(q.astype(np.longdouble) - ref)))
    top = float(ref[-1])
    assert err <= TABLE_TOL * top, (len(x), err, top)
    return err / top if top else 0.0


def addressed_signals(rng, n_max):
    """Rows of one (6, T) tensor with odd T, slices at storage offsets 1, 2 and 3 (NaN around them) and one signal 8
    times longer; all finite."""
    T = n_max + 1 + (n_max % 2)                               # odd
    rows = torch.from_numpy(np.stack([dry_signal(KINDS[j % 3], rng, T) for j in range(6)])).cuda()
    sig = list(rows.unbind(0))
    for o in (1, 2, 3):
        base = torch.full((n_max + 8,), NAN, device="cuda")
        base[o:o + n_max] = to(dry_signal(KINDS[o % 3], rng, n_max))
        sig.append(base[o:o + n_max])
    sig.append(to(so.synth_dry(rng, 8 * n_max + 3)))
    return sig


def test_signal_addressing():
    render, R = _R()
    rng = np.random.default_rng(1201)
    grid, aligned = DevPool(a_grid(rng)), DevPool(a_aligned(rng), taps=TAPS)
    n_max = max(grid.n_max, aligned.n_max)
    sig_d = addressed_signals(rng, n_max)
    assert {x.data_ptr() % 16 for x in sig_d[:6]} == {0, 4, 8, 12}
    assert [x.storage_offset() for x in sig_d[6:9]] == [1, 2, 3]
    sig_h = [x.cpu().numpy() for x in sig_d]
    dp = R.dry_pool(sig_d, levels=True)
    slots = [DrySlots(pl, dp, [3001, 64000], 6) for pl in (grid, aligned)]
    try:
        worst = 0.0
        for i, x in enumerate(sig_h):
            worst = max(worst, table_check(dp.level_table(i).cpu().numpy(), x))
        jobs = []
        for sl, pl, name in zip(slots, (grid, aligned), ("grid", "aligned")):
            n = len(sl.slots)
            snaps, vals = [], []
            for r in range(3):                                # every signal, at random starts
                v = np.zeros((3, n), np.int32)
                for j, wl in enumerate(sl.slots):
                    i = int(rng.integers(0, len(pl.cands)))
                    v[:, j] = i, (r * n + j) % dp.n, int(rng.integers(0, pl.cands[i].N - wl)) | 1
                vals.append(v)
                snaps.append(sl.run(to(v)))
            assert {int(d) for v in vals for d in v[1]} == set(range(dp.n))
            R.check_device_errors()
            for r in range(3):
                sl.check(vals[r], snaps[r], sig_d, sig_h, "B %s" % name, "addressing %s run %d" % (name, r), jobs)
        check_f64(jobs)
        print("\naddressing: worst table error %.3g x TABLE_TOL" % (worst / TABLE_TOL))
        _report("B")
    finally:
        for sl in slots:
            sl.close()
        dp.close()
        grid.close()
        aligned.close()


# ----------------------------------------------------------------------------------------- C. multi-chunk plans
C_WL = 1500
C_KINDS = ["dry aligned", "plain grid", "dry long", "unpooled", "dry grid", "plain aligned", "dry aligned",
           "plain long", "static", "dry grid"]


def c_pools(rng):
    aligned = [ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, B), np.round(np.linspace(0, N, P)).astype(np.int32))
               for N, P in ((20001, 3), (24002, 4), (28003, 3))]
    assert all(_choice(c.b, c.N, c.P, B) == 1 for c in aligned)
    grid = []
    for j, N in enumerate((22001, 25003)):
        np.random.seed(530 + j)
        b = _bounds_of(so.setup_dynamic_interp(so.synth_path(rng, 30), N)[0], 30)
        assert _choice(b, N, 30, B) == 0
        grid.append(ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, 30, 2, B), b))
    longs = [ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, 3, 2, L), _random_cuts(rng, 3, N))
             for N, L in ((21001, 9000), (26002, 12288))]
    return {"aligned": DevPool(aligned), "grid": DevPool(grid), "long": DevPool(longs)}


class BigPlan:
    """Slots in caller order cycling C_KINDS: dry-picked slots alternate between two dry pools; unpooled banked moving
    sources and a static source at fixed windows."""

    def __init__(self, pools, dps, extra, n):
        render, R = _R()
        self.kinds = [C_KINDS[j % len(C_KINDS)] for j in range(n)]
        self.vals = torch.zeros((3, n), dtype=torch.int32, device="cuda")
        self.pools, self.dps, self.extra = pools, dps, extra
        srcs, self.fixed = [], {}
        for j, k in enumerate(self.kinds):
            if k in ("unpooled", "static"):
                c, src = extra[k]
                s = (37 * j) % (c.N - C_WL + 1)
                self.fixed[j] = s
                srcs.append(src._replace(window=(s, C_WL)))
                continue
            pl = pools[k.split()[1]]
            dry = render.DryPick(dps[j % 2], self.vals[1, j]) if k.startswith("dry") else None
            srcs.append(render.Pooled(pl.pool, self.vals[0, j], (self.vals[2, j], C_WL), 0, dry))
        self.outs = [Out(2, C_WL) for _ in range(n)]
        self.plan = R.plan_device(srcs, [o.view() for o in self.outs])

    def values(self, rng):
        n = len(self.kinds)
        v = np.zeros((3, n), np.int32)
        for j, k in enumerate(self.kinds):
            if j in self.fixed:
                continue
            pl = self.pools[k.split()[1]]
            i = int(rng.integers(0, len(pl.cands)))
            v[:, j] = i, int(rng.integers(0, self.dps[j % 2].n)), int(rng.integers(0, pl.cands[i].N - C_WL + 1))
        return v

    def run(self, v):
        for o in self.outs:
            o.reset()
        self.vals.copy_(v)
        self.plan.run()
        return [o.buf.clone() for o in self.outs]

    def check(self, v, snap, sig, jobs, label):
        for j, k in enumerate(self.kinds):
            y = self.outs[j].get(snap[j])
            what = "%s slot %d (%s)" % (label, j, k)
            if j in self.fixed:
                c, src = self.extra[k]
                s = self.fixed[j]
                out = torch.empty((2, C_WL), device="cuda")
                _R()[1].render_device([src._replace(window=(s, C_WL))], [out])
                assert np.array_equal(y, out.cpu().numpy()), what
                jobs.append(("C %s" % k, what, c.x, c, s, C_WL, y, False))
                continue
            pl = self.pools[k.split()[1]]
            i, d, s = (int(a) for a in v[:, j])
            xd, xh = sig[j % 2][0][d], sig[j % 2][1][d]
            if k.startswith("plain"):
                xd = xh = None
            check_stem(pl, i, xd, xh, s, C_WL, y, None, "C %s" % k, what + " cand %d dry %d start %d" % (i, d, s),
                       jobs)

    def close(self):
        self.plan.close()


def test_multi_chunk_plan_over_two_dry_pools(chunk_budget):
    render, R = _R()
    rng = np.random.default_rng(1301)
    pools = c_pools(rng)
    n_max = max(p.n_max for p in pools.values())
    sig = [dry_set(rng, n_max, 6), dry_set(rng, n_max + 11, 5, tails=(0, 3, 1, 2, 9))]
    sig = [(d, h) for h, d in sig]
    dps = [R.dry_pool(sig[0][0]), R.dry_pool(sig[1][0])]
    ext = [ScaleCand(so.synth_dry(rng, 30001), so.synth_rirs(rng, 4, 2, 6000), np.array([0, 9000, 20000, 30001], np.int32)),
           ScaleCand(so.synth_dry(rng, 27001), so.synth_rirs(rng, 1, 2, 3000), None)]
    banks = [R.rir_bank(to(ext[0].h)), R.rir_bank(to(ext[1].h[0]))]
    extra = {"unpooled": (ext[0], render.MovingSource(to(ext[0].x), banks[0], to(ext[0].b), ext[0].b)),
             "static": (ext[1], render.StaticSource(to(ext[1].x), banks[1]))}
    n = 1040
    plans, ref = [], None
    try:
        v = None
        counts = {}
        for budget in (DEFAULT_CHUNK_BYTES, 2 << 20):
            chunk_budget(budget)
            bp = BigPlan(pools, dps, extra, n)
            plans.append(bp)
            if v is None:
                v = bp.values(rng)
            dv = to(v)
            R.reset_stats()
            snap = bp.run(dv)
            counts[budget] = R.launch_count()
            torch.cuda.synchronize()
            R.check_device_errors()
            if ref is None:                                   # every stem: render_device and float64
                jobs = []
                bp.check(v, snap, sig, jobs, "default budget")
                check_f64(jobs)
                ref = [bp.outs[j].get(snap[j]).copy() for j in range(n)]
            else:                                             # the same bits in many chunks
                for j in range(n):
                    assert np.array_equal(bp.outs[j].get(snap[j]), ref[j]), ("small budget", j, bp.kinds[j])
        print("\n1040 slots: launches per run %s (default, 2 MB budget)" % list(counts.values()))
        assert counts[2 << 20] > counts[DEFAULT_CHUNK_BYTES] + 30, counts
        # a second plan over the first dry pool, run in turn with the first on the same stream
        small = DrySlots(pools["aligned"], dps[0], [C_WL, 5000], 4)
        plans.append(small)
        v2 = np.zeros((3, len(small.slots)), np.int32)
        for j, wl in enumerate(small.slots):
            i = j % 3
            v2[:, j] = i, (5 - j) % dps[0].n, (97 * j) % (pools["aligned"].cands[i].N - wl + 1)
        s1 = plans[1].run(to(v))
        s2 = small.run(to(v2))
        s3 = plans[1].run(to(v))
        torch.cuda.synchronize()
        jobs = []
        small.check(v2, s2, sig[0][0], sig[0][1], "C second plan", "second plan", jobs)
        check_f64(jobs)
        for s in (s1, s3):
            for j in range(n):
                assert np.array_equal(plans[1].outs[j].get(s[j]), ref[j]), ("in turn", j)
        R.check_device_errors()
        _report("C")
    finally:
        for p in plans:
            p.close()
        for d in dps:
            d.close()
        for p in pools.values():
            p.close()
        for b in banks:
            b.close()


# ----------------------------------------------------------------------------------------- D. draws
@pytest.fixture(scope="module")
def dry_beacons():
    """Speaker lane ("spk", i) of test_gpu_pool_builds.Case is a slot of the trajectory pool (candidate 0 of NS samples
    for i < 2, else candidate 1 of NL) that picks dry signal i - zoned with its end zone at NS (0), loud (1, 3), zoned
    with its end zone at NL (2) - or, for a loud speaker marked plain, no dry signal; ("noi", i) a slot of a noise pool
    (NL, NN).  So the designed M, starts and outcomes of Case hold unchanged."""
    render, R = _R()
    rng = np.random.default_rng(1401)
    tp = DevPool([traj_beacon(rng, NS), traj_beacon(rng, NL)], levels="mono")
    npl = DevPool([traj_beacon(rng, NL), traj_beacon(rng, NN)])
    dry_h = [dry_beacon(rng, NL, NS), dry_beacon(rng, NL, 0), dry_beacon(rng, NL, NL), dry_beacon(rng, NL, 0)]
    dry_d = [to(x) for x in dry_h]
    dp = R.dry_pool(dry_d, levels=True)
    bw = type("Beacons", (), {})()
    bw.tp, bw.np, bw.dp, bw.dry_d = tp, npl, dp, dry_d
    bw.Td = [dp.level_table(i).cpu().numpy() for i in range(dp.n)]
    bw.Tp = [tp.pool.level_table(i).cpu().numpy() for i in range(2)]
    full = {}
    for i in range(4):                                         # whole stems: dry-picked, plain, noise
        c = tp.cands[0 if i < 2 else 1]
        full[("dry", i)] = torch.from_numpy(tp.ref(0 if i < 2 else 1, dry_d[i], 0, c.N)[0]).cuda()
    for t in range(2):
        full[("plain", t)] = torch.from_numpy(tp.ref(t, None, 0, tp.cands[t].N)[0]).cuda()
        full[("noi", t)] = torch.from_numpy(npl.ref(t, None, 0, npl.cands[t].N)[0]).cuda()
    bw.full = full
    yield bw
    for p in (tp, npl):
        p.close()
    dp.close()


def test_draw_warp_edges_with_dry_speakers(dry_beacons):
    render, R = _R()
    bw = dry_beacons
    large = d_cases(LARGE)
    small = d_cases(SMALL, seeds=range(5))[:997]              # 997 = 4 * 249 + 1: the last CTA holds one draw
    chunks, at = [], 0
    for n in (1, 3, 4, 5):
        chunks.append(large[at:at + n])
        at += n
    while at < len(large):
        chunks.append(large[at:at + 50])
        at += 50
    chunks.append(small)
    assert len(small) == 997
    _device_errors(R)
    outcomes, worst, dry_hi = set(), np.inf, 0
    for n, ch in enumerate(chunks):
        dp = DryDrawPlan(bw, ch)
        try:
            dp.run()
            assert _device_errors(R) == 0, n
            worst = min(worst, dp.check(bw, "plan %d of %d draws" % (n, len(ch))))
            assert dp.plan.is_graph()
            dry_hi += sum(1 for c, w in zip(ch, dp.what) for lane in c.speakers if lane >= 8 and w[lane][0] == "dry")
        finally:
            dp.close()
        outcomes |= {(c.tries, c.tstar) for c in ch}
    assert outcomes == set(d_combos())
    assert dry_hi >= 100, dry_hi                               # dry-picked speakers at reader lanes 8 to 15
    print("\ndry warp edges: %d draws in %d plans, least margin %.1f dB, %d dry-picked speakers at lanes >= 8"
          % (len(large) + len(small), len(chunks), worst, dry_hi))


def test_training_plan_of_dry_picked_examples():
    """64 examples x (2 dry-picked speakers + a dry-picked noise), 4 s crops drawn over the dry pool's tables, one mono
    mixture each: stems against render_device, mixtures against mix_reference, draws against draw_reference."""
    render, R = _R()
    rng = np.random.default_rng(1402)
    spk = DevPool([ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, B), np.round(np.linspace(0, N, P)).astype(np.int32))
                   for N, P in ((150001, 4), (160002, 5), (170003, 6), (155004, 4), (165005, 5), (175006, 3))])
    noi = DevPool([ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 2048), None) for N in (160001, 170002, 180003)])
    n_max = max(spk.n_max, noi.n_max)
    dry_h = [gappy_dry(rng, n_max + 1000 * j) for j in range(24)]
    dry_d = [to(x) for x in dry_h]
    dp = R.dry_pool(dry_d, levels=True)
    Td = [dp.level_table(i).cpu().numpy() for i in range(dp.n)]
    U, T = 64, 4 * RATE
    picks = torch.zeros((U, 3), dtype=torch.int32, device="cuda")
    dpicks = torch.zeros((U, 3), dtype=torch.int32, device="cuda")
    starts = torch.zeros(U, dtype=torch.int32, device="cuda")
    u = torch.zeros((U, 101), dtype=torch.float64, device="cuda")
    used = torch.zeros(U, dtype=torch.int32, device="cuda")
    sirs, snr = torch.zeros((U, 1), device="cuda"), torch.zeros(U, device="cuda")
    outs = [Out(2, T) for _ in range(3 * U)]
    mix, spo, rms = [Out(1, T) for _ in range(U)], [Out(2, T) for _ in range(U)], [Out(1, 2) for _ in range(U)]
    srcs, mixes, draws = [], [], []
    for e in range(U):
        for k, pl in enumerate((spk, spk, noi)):
            srcs.append(render.Pooled(pl.pool, picks[e, k], (starts[e], T), 0, render.DryPick(dp, dpicks[e, k])))
        mixes.append(render.Mixture([3 * e, 3 * e + 1], [3 * e + 2], sirs[e], snr[e], mix[e].view(T),
                                    spo[e].view(2, T), rms[e].view(2), mono=True))
        draws.append(render.CropDraw(starts[e], [3 * e, 3 * e + 1], u[e], used[e]))
    plan = R.plan_device(srcs, [o.view() for o in outs], mixtures=mixes, draws=draws)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1403)
    checked = near = 0
    try:
        for run in range(2):
            for o in outs + mix + spo + rms:
                o.reset()
            picks[:, :2].copy_(torch.randint(0, len(spk.cands), (U, 2), generator=gen, device="cuda", dtype=torch.int32))
            picks[:, 2].copy_(torch.randint(0, len(noi.cands), (U,), generator=gen, device="cuda", dtype=torch.int32))
            dpicks.copy_(torch.randint(0, dp.n, (U, 3), generator=gen, device="cuda", dtype=torch.int32))
            u.uniform_(generator=gen)
            sirs.uniform_(-6, 6, generator=gen)
            snr.uniform_(10, 20, generator=gen)
            plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            pk, dk, st = picks.cpu().numpy(), dpicks.cpu().numpy(), starts.cpu().numpy()
            us, ud = u.cpu().numpy(), used.cpu().numpy()
            for e in range(U):
                s = int(st[e])
                stems = []
                for k, pl in enumerate((spk, spk, noi)):
                    y = outs[3 * e + k].get()
                    ref, _ = pl.ref(int(pk[e, k]), dry_d[dk[e, k]], s, T)
                    assert np.array_equal(y, ref), (run, e, k)
                    stems.append(y)
                check_mixture(np.stack([fold(a) for a in stems[:2]]), fold(stems[2])[None], sirs[e].cpu().numpy(),
                              snr[e].cpu().numpy(), mix[e].get().reshape(-1), spo[e].get().reshape(2, -1),
                              rms[e].get().reshape(-1), "training run %d example %d" % (run, e))
                tabs = [Td[dk[e, 0]], Td[dk[e, 1]]]
                Nr = [spk.cands[pk[e, 0]].N, spk.cands[pk[e, 1]].N, noi.cands[pk[e, 2]].N]
                if dr.margins(tabs, [T, T], Nr, T, us[e]) < NEAR_DB:
                    near += 1
                    continue
                assert (s, int(ud[e])) == dr.draw(tabs, [T, T], Nr, T, us[e]), (run, e)
                checked += 1
        assert plan.is_graph()
        print("\ntraining plan: %d draws checked, %d near the threshold" % (checked, near))
        assert checked >= 120 and near <= 4, (checked, near)
    finally:
        plan.close()
        dp.close()
        spk.close()
        noi.close()


# ----------------------------------------------------------------------------------------- E. dry pool builds
TILE = 2048                      # samples of one k_levels tile (256 threads x 8)
E_LENS = sorted({1, 2} | {TILE * k + d for k in range(1, 9) for d in (-1, 0, 1)} | {2 * TILE * k + d for k in (1, 2)
                                                                                        for d in (-1, 0, 1)})
N_BIG = 65537 + 5


def _tables_of(dp, lens):
    """Every table of a dry pool in one copy: tables lie back to back (N + 1 doubles each) from table 0 on."""
    total = int(sum(n + 1 for n in lens))
    ptr = dp.renderer.lib.ss_dry_pool_level_table(dp._h, 0)
    for i in (1, len(lens) - 1):
        assert dp.renderer.lib.ss_dry_pool_level_table(dp._h, i) == ptr + 8 * int(sum(n + 1 for n in lens[:i]))

    class _View:
        __cuda_array_interface__ = {"shape": (total,), "typestr": "<f8", "data": (ptr, False), "version": 3}
    return torch.as_tensor(_View(), device="cuda").clone().cpu().numpy()


def test_level_tables_at_tile_edges_and_alignments():
    _, R = _R()
    rng = np.random.default_rng(1501)
    lens = E_LENS + [3 * TILE + 5, 1]
    base = torch.full((sum(lens) + 8 * len(lens) + 16,), NAN, device="cuda")
    sig, at = [], 0
    for j, n in enumerate(lens):
        at += j % 4                                            # 4-, 8- and 12-byte alignments
        x = so.synth_dry(rng, n) * np.float32(1 + j % 5)
        if j == len(E_LENS):                                   # all-zero signal
            x[:] = 0.0
        base[at:at + n] = to(x)
        sig.append(base[at:at + n])
        at += n + 3
    assert {x.data_ptr() % 16 for x in sig} == {0, 4, 8, 12}
    host = [x.cpu().numpy() for x in sig]
    a, b = R.dry_pool(sig, levels=True), R.dry_pool(sig, levels=True)
    try:
        assert a.nbytes == 8 * a.n + 8 * sum(len(x) + 1 for x in host) + 8 * a.n
        worst = 0.0
        for i, x in enumerate(host):
            q = a.level_table(i)
            assert torch.equal(q, b.level_table(i)), len(x)
            worst = max(worst, table_check(q.cpu().numpy(), x))
        assert not a.level_table(len(host) - 2).cpu().numpy().any()      # all zero: exactly 0
        print("\ntile edges: %d signals, worst table error %.3g x TABLE_TOL" % (len(host), worst / TABLE_TOL))
    finally:
        a.close()
        b.close()


def test_pool_past_one_levels_launch():
    """65 542 short signals, views of one tensor: two k_levels launches, every table against the long-double prefix,
    the same bits again, and picks at indices >= 65 535 rendered and drawn in a plan."""
    render, R = _R()
    rng = np.random.default_rng(1502)
    lens = rng.integers(48, 72, N_BIG).astype(np.int64)
    m = int(lens.sum())                                        # samples of magnitude 0.5 to 1: no crop near -40 dB
    flat_h = (rng.choice([-1.0, 1.0], m) * (0.5 + 0.5 * rng.random(m))).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(lens)])
    for i in range(65530, 65542, 2):                           # silent heads around index 65 535: starts <= 8 silent
        flat_h[off[i]:off[i] + 24] = 0.0
    flat = to(flat_h)
    sig = [flat[int(off[i]):int(off[i + 1])] for i in range(N_BIG)]
    # the library's own launch count: a dry pool build launches k_levels and nothing else.  (A torch.profiler session
    # here would open the process's first CUPTI session, and test_gpu_pool_builds' per-kernel counts, which run later
    # in the suite, have been seen to drop a kernel record in a session that is not the process's first.)
    torch.cuda.synchronize()
    R.reset_stats()
    dp = R.dry_pool(sig, levels=True)
    assert R.launch_count() == 2
    again = R.dry_pool(sig, levels=True)
    tp = DevPool([ScaleCand(so.synth_dry(rng, 40), so.synth_rirs(rng, 1, 1, 8), None),
                  ScaleCand(so.synth_dry(rng, 48), so.synth_rirs(rng, 1, 1, 8), None)], levels="mono")
    try:
        assert dp.nbytes == 8 * N_BIG + 8 * int((lens + 1).sum()) + 8 * N_BIG
        q = _tables_of(dp, lens)
        assert np.array_equal(q, _tables_of(again, lens))
        e = (flat_h.astype(np.float32) ** 2).astype(np.longdouble)
        worst = 0.0
        for i in range(N_BIG):                                 # every table, both launches
            t = q[off[i] + i:off[i + 1] + i + 1]
            ref = np.concatenate([[0.0], np.cumsum(e[off[i]:off[i + 1]])])
            assert t[0] == 0.0
            err = float(np.max(np.abs(t.astype(np.longdouble) - ref)))
            assert err <= TABLE_TOL * float(ref[-1]), (i, err)
            worst = max(worst, err / float(ref[-1]))
        # picks at 65 533 .. 65 541 in a plan: stems and draws
        wl, n = 16, 9
        vals = torch.zeros((3, n), dtype=torch.int32, device="cuda")
        used = torch.zeros(n, dtype=torch.int32, device="cuda")
        uh = rng.random((n, 7))
        uh[:, :2] = 0.1, 0.9                                   # starts 2 (silent in a silent head) and 22
        u = to(uh)
        outs = [Out(1, wl) for _ in range(n)]
        srcs = [render.Pooled(tp.pool, vals[0, j], (vals[2, j], wl), 0, render.DryPick(dp, vals[1, j]))
                for j in range(n)]
        draws = [render.CropDraw(vals[2, j], [j], u[j], used[j]) for j in range(n)]
        plan = R.plan_device(srcs, [o.view() for o in outs], draws=draws)
        try:
            v = np.array([[j % 2 for j in range(n)], [65533 + j for j in range(n)], [0] * n], np.int32)
            vals.copy_(to(v))
            plan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            st, us, ud = vals[2].cpu().numpy(), u.cpu().numpy(), used.cpu().numpy()
            jobs, firsts = [], set()
            for j in range(n):
                i, d, s = int(v[0, j]), int(v[1, j]), int(st[j])
                check_stem(tp, i, sig[d], flat_h[off[d]:off[d + 1]], s, wl, outs[j].get(), None, "E past one launch",
                           "signal %d" % d, jobs)
                tab = q[off[d] + d:off[d + 1] + d + 1]
                Nr = [tp.cands[i].N]
                assert dr.margins([tab], [wl], Nr, wl, us[j]) >= NEAR_DB, j
                assert (s, int(ud[j])) == dr.draw([tab], [wl], Nr, wl, us[j]), j
                firsts.add(int(ud[j]) == 1)
            check_f64(jobs)
            assert firsts == {True, False}, firsts
        finally:
            plan.close()
        print("\n%d signals: 2 k_levels launches, worst table error %.3g x TABLE_TOL" % (N_BIG, worst / TABLE_TOL))
    finally:
        dp.close()
        again.close()
        tp.close()


# ----------------------------------------------------------------------------------------- F. lifetimes
def test_dry_pool_closed_under_live_plans():
    render, R = _R()
    rng = np.random.default_rng(1601)
    pl = DevPool(a_aligned(rng))
    n_sig, T = 8, 1700000                                      # 8 x 1.7 M samples: 109 MB of level tables
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    sig = [to(gappy_dry(rng, T)) for _ in range(n_sig)]
    host = [x.cpu().numpy() for x in sig]
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    dp = R.dry_pool(sig, levels=True)
    torch.cuda.synchronize()
    free2 = torch.cuda.mem_get_info()[0]
    assert dp.nbytes >= 100e6 and free1 - free2 >= 0.95 * dp.nbytes, (dp.nbytes, free1 - free2)
    slots = [DrySlots(pl, dp, [5000, 3001], 3), DrySlots(pl, dp, [64000], 2)]
    vals = []
    for sl in slots:
        v = np.zeros((3, len(sl.slots)), np.int32)
        for j, wl in enumerate(sl.slots):
            i = int(rng.integers(0, len(pl.cands)))
            v[:, j] = i, int(rng.integers(0, n_sig)), int(rng.integers(0, pl.cands[i].N - wl + 1))
        vals.append(v)
    try:
        jobs, before = [], []
        for sl, v in zip(slots, vals):
            snap = sl.run(to(v))
            torch.cuda.synchronize()
            sl.check(v, snap, sig, host, "F", "before close", jobs)
            before.append([o.get(s).copy() for o, s in zip(sl.outs, snap)])
        check_f64(jobs)
        dp.close()
        assert dp.closed
        with pytest.raises(ValueError, match="is closed"):
            R.plan_device([render.Pooled(pl.pool, slots[0].vals[0, 0], (slots[0].vals[2, 0], 5000), 0,
                                         render.DryPick(dp, slots[0].vals[1, 0]))], [torch.empty((2, 5000), device="cuda")])
        del sig
        gc.collect()
        junk = [torch.full((T,), 7.0, device="cuda") for _ in range(n_sig)]
        for _ in range(2):
            for sl, v, ref in zip(slots, vals, before):
                snap = sl.run(to(v))
                torch.cuda.synchronize()
                for o, s, r in zip(sl.outs, snap, ref):
                    assert np.array_equal(o.get(s), r)
        R.check_device_errors()
        del junk
        torch.cuda.synchronize()
        free3 = torch.cuda.mem_get_info()[0]
        slots[0].close()
        torch.cuda.synchronize()
        assert torch.cuda.mem_get_info()[0] - free3 < 0.5 * dp.nbytes         # still held by the second plan
        slots[1].close()
        gc.collect()
        torch.cuda.synchronize()
        free4 = torch.cuda.mem_get_info()[0]
        assert free4 - free3 >= 0.95 * dp.nbytes, (dp.nbytes, free4 - free3)  # returned after the last plan
        print("\nlifetimes: %.1f MB of dry pool returned after the last plan closed (free %d -> %d -> %d bytes)"
              % (dp.nbytes / 1e6, free0, free3, free4))
        _report("F")
    finally:
        for sl in slots:
            sl.close()
        dp.close()
        pl.close()
