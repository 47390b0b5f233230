"""Level tables, loudness gains and start draws of source pools at training scale, through the real kernels.

ss_pool_loudness and ss_pool_levels render a pool's candidates whole into one transient buffer, in groups of
consecutive candidates that fit 256 MiB (a larger candidate is a group of its own and the buffer grows to fit it); a
training pool (64 configs[1] scenes) always has several groups.  k_draw runs the dataloader's start loop one warp per
draw: a min-reduction of M over up to 16 readers, up to 8 speaker tables, rounds of 32 tries with a ballot, and the last
try's start from the last round.  Checked:
  A. a moving pool of 48 configs[1] speakers (3 groups) and a static 8-channel pool with one candidate larger than
     256 MiB between ordinary ones (groups [3], [giant], [3]):
       - the group boundaries restated from the grouping rule, and reached: k_levels and k_loud_scale launch once per
         group (torch.profiler);
       - for every candidate, mono and channel tables: SourcePool.loudness equals render_host(..., lufs_targets=) of the
         candidate alone bit for bit and the float64 BS.1770 oracle within 1e-6 dB; its table is within TABLE_TOL * Q[N]
         of the long-double prefix of that normalised stem; a second build and a one-candidate pool give the same bits;
         unmeasured and silent candidates sit at group edges and on each side of the giant;
       - render_host stems at the first and last candidate of every group and windows of the giant against float64;
       - a training plan over the normalised multi-group pool: draws against draw_reference on float64 tables of the
         render_host stems, crops bit for bit, mixtures against ss_mix_dev;
  B. beacon pools (loud everywhere except silent zones, so every try's outcome is known by tens of dB): every tries in
     {1, 2, 31, 32, 33, 63, 64, 65, 101, 4095, 4096} with the first passing try at 0, 1, 30, 31, 32, 33, 63, 64,
     tries - 1 or none; 1 to 16 readers with the shortest at lane 0, lane 15, a middle lane or a noise reader of another
     pool; 1 to 8 speakers with the silent one at speaker 0, 7 or between; u of 0, 1 - 2^-53, 1, < 0 and NaN in a second
     round; plans of 1, 3, 4, 5 and about 1000 draws; an out-of-range pick (clamped, bit 3 alone).  Every start and
     `used` equals both the design and draw_reference, and every reader's crop the slice of its whole stem;
  C. k_levels tile edges: N from 1 to 2048 k + 1 around the 2048-sample tiles, C in {1, 3, 5, 8}, a silent stretch of
     whole tiles, both table kinds, against the long-double prefix."""
import types

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
import draw_reference as dr
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from draw_reference import Step, TABLE_TOL, check_snap, gappy_dry
from gpu_plumbing import _R, _device_errors
from pool_worlds import (Cand, Case, EDGE, LARGE, LB, NL, NN, NS, SMALL, STEM_BYTES, TSTARS, WB, Z0, Z1, _mix_dev,
                         align_up, fold_dev, host_src, stem_groups, table_error)

pytestmark = pytest.mark.gpu

RATE = 16000
NAN = float("nan")


def host_stem(R, render, c, target=None):
    """render_host of the candidate alone: its (C, N) stem and, with a target, the (LUFS, gain) it measured."""
    lo = []
    y = R.render_host([host_src(render, c)], lufs_targets=None if target is None else [target], loudness_out=lo,
                      sr=RATE)[0]
    return y, (tuple(lo[0]) if target is not None else None)


def launches(prof, name):
    return sum(1 for e in prof.events() if name in e.name)


# ----------------------------------------------------------------------------------------- A. stem groups
class Big:
    """A pool's candidates, targets, restated groups, and per candidate the render_host references: the normalised
    stem (the raw one without a target), the (LUFS, gain) it measured and the float64 oracle's LUFS of the raw stem."""

    def __init__(self, kind):
        render, R = _R()
        if kind == "moving":
            import bench
            C, N = bench.CFG["C"], bench.CFG["N"]
            items = bench.make_inputs(24, 0)                     # 48 configs[1] speakers: C = 6, P = 40, L = 4096
            cut = {5: 1, 21: 7, 30: 13, 47: 29}                  # 4 C N not a multiple of 256
            Ns = [N - cut.get(j, 0) for j in range(len(items))]
            self.first, self.cap = stem_groups(C, Ns)
            assert self.first == [0, 23, 46, 48], self.first
            unmeasured = {self.first[1], self.first[2] - 1, self.first[2]}
            silent = {self.first[1] - 1}
            rng = np.random.default_rng(301)
            cands = []
            for j, ((x, h, b), n) in enumerate(zip(items, Ns)):
                x = (gappy_dry(rng, n) * np.float32(4.0)) if j % 2 else x[:n].copy()
                b = b.copy()
                b[-1] = n
                if j in silent:
                    x[:] = 0.0
                cands.append(Cand(x, h, b))
        else:
            rng = np.random.default_rng(302)
            Ns = [300000 + 7 * j for j in range(3)] + [8500003] + [310001 + 5 * j for j in range(3)]
            self.first, self.cap = stem_groups(8, Ns)
            assert self.first == [0, 3, 4, 7] and self.cap == align_up(4 * 8 * 8500003, 256) > STEM_BYTES, self.first
            unmeasured, silent = {2}, {4}                        # on each side of the giant
            cands = []
            for j, n in enumerate(Ns):
                x = so.synth_dry(rng, n) * np.float32(0.5 + 0.25 * (j % 3))
                if j in silent:
                    x[:] = 0.0
                cands.append(Cand(x, so.synth_rirs(rng, 1, 8, 1024)[0], None))
        self.kind, self.cands, self.C = kind, cands, cands[0].C
        self.silent = silent
        trng = np.random.default_rng(303)
        self.targets = [None if j in unmeasured else float(trng.uniform(-30, -14)) for j in range(len(cands))]
        self.norm, self.loud, self.oracle = [], [], []
        for c, t in zip(cands, self.targets):
            raw, _ = host_stem(R, render, c)
            if t is None:
                self.norm.append(raw)
                self.loud.append(None)
                self.oracle.append(None)
                continue
            y, lo = host_stem(R, render, c, t)
            self.norm.append(y)
            self.loud.append(lo)
            self.oracle.append(so.bs1770_integrated_loudness(raw.T.astype(np.float64), RATE, 0.4,
                                                             up_to_8_channels=True))

    def groups(self):
        return [(self.first[g], self.first[g + 1]) for g in range(len(self.first) - 1)]


@pytest.fixture(scope="module", params=["moving", "static"])
def big(request):
    w = Big(request.param)
    yield w
    del w
    torch.cuda.empty_cache()


@pytest.mark.parametrize("levels", ["mono", "channels"])
def test_tables_and_gains_across_groups(big, levels):
    render, R = _R()
    mono = levels == "mono"
    srcs = [c.src for c in big.cands]
    G = big.groups()
    measured = sum(1 for a, b in G if any(t is not None for t in big.targets[a:b]))
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        a = R.source_pool(srcs, levels=levels, lufs_targets=big.targets, sr=RATE)
        torch.cuda.synchronize()
    counts = {k: launches(prof, k) for k in ("k_levels", "k_loud_scale", "k_loud_gate")}
    print("%s %s: groups %s, launches %s" % (big.kind, levels, big.first, counts))
    assert counts == {"k_levels": len(G), "k_loud_scale": len(G), "k_loud_gate": measured}, (counts, big.first)
    b = R.source_pool(srcs, levels=levels, lufs_targets=big.targets, sr=RATE)
    worst_tab = worst_db = 0.0
    try:
        La, Lb = a.loudness, b.loudness
        assert La.tobytes() == Lb.tobytes()
        for i, (c, t) in enumerate(zip(big.cands, big.targets)):
            what = (big.kind, levels, i)
            q = a.level_table(i)
            assert torch.equal(q, b.level_table(i)), what
            one = R.source_pool([c.src], levels=levels, lufs_targets=[t], sr=RATE)
            try:
                assert torch.equal(one.level_table(0), q), what                # bits that depend on N alone
                assert one.loudness.tobytes() == La[i:i + 1].tobytes(), what
            finally:
                one.close()
            if t is None:
                assert np.isnan(La[i]).all(), what
            else:
                assert (La[i, 0], La[i, 1]) == big.loud[i], (what, La[i], big.loud[i])           # -inf == -inf
                if i in big.silent:
                    assert np.isneginf(La[i, 0]) and np.isneginf(big.oracle[i]), what
                    assert La[i, 1] == pytest.approx(10.0 ** ((t + 40.0) / 20.0), rel=1e-15), what
                else:
                    d = abs(La[i, 0] - big.oracle[i])
                    assert d < 1e-6, (what, La[i, 0], big.oracle[i])
                    worst_db = max(worst_db, d)
            r = table_error(q.cpu().numpy(), big.norm[i], mono)
            assert r <= TABLE_TOL, (what, r / TABLE_TOL)
            worst_tab = max(worst_tab, r)
        print("%s %s: worst table error %.3g x TABLE_TOL, worst loudness vs the oracle %.3g dB"
              % (big.kind, levels, worst_tab / TABLE_TOL, worst_db))
    finally:
        a.close()
        b.close()


def test_renders_at_group_edges(big):
    """The render_host stems the tables and gains are checked against, sample by sample against float64 (times the
    float32 gain the stem carries): the first and last candidate of every group, and windows of the giant."""
    wl = 8192
    worst = 0.0
    for a, b in big.groups():
        for i in sorted({a, b - 1}):
            c = big.cands[i]
            g = float(np.float32(big.loud[i][1])) if big.loud[i] is not None else 1.0
            wins = [0, c.N - wl] if c.N < 1000000 else [0, c.N // 2 - 3001, c.N - wl]
            for s in wins:
                y64, scale = render_check_inputs(c.x, c.h, 0 if c.b is None else 1, bounds=c.b, window=(s, wl))
                r, _ = check_render(big.norm[i][:, s:s + wl], y64 * g, scale * g, TAU_LOCAL, TAU_GLOBAL, n0=s,
                                    label="%s candidate %d window %d" % (big.kind, i, s))
                worst = max(worst, r)
    print("%s: worst local render error %.3g" % (big.kind, worst))


@pytest.mark.parametrize("big", ["moving"], indirect=True)
def test_draws_over_a_multi_group_pool(big):
    """16 examples over 4 runs, both speakers of every example forced into chosen groups (every group's first and last
    candidate included): draws against draw_reference on float64 tables of the render_host stems."""
    render, R = _R()
    rng = np.random.default_rng(304)
    noi = [Cand(so.synth_dry(rng, 470000 + 1001 * j), so.synth_rirs(rng, 1, big.C, 2048)[0], None) for j in range(3)]
    nnoi = [types.SimpleNamespace(N=c.N, full=torch.from_numpy(host_stem(R, render, c)[0]).cuda()) for c in noi]
    nspk = [types.SimpleNamespace(N=c.N, full=torch.from_numpy(y).cuda()) for c, y in zip(big.cands, big.norm)]
    Ts = [dr.level_table(y, True) for y in big.norm]
    sm = R.source_pool([c.src for c in big.cands], levels="mono", lufs_targets=big.targets, sr=RATE)
    npool = R.source_pool([c.src for c in noi])
    st = Step(R, render, sm, npool, B=16)
    LEN = st.outs[0].shape[1]
    G = big.groups()
    edges = sorted({i for a, b in G for i in (a, b - 1)})
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5)
    total = near = 0
    seen = set()
    try:
        for run in range(4):
            st.fill(gen, len(big.cands), len(noi))
            pk = np.zeros((16, 2), np.int32)
            for b in range(16):
                a0, a1 = G[(b + run) % len(G)]
                pk[b] = (edges[(16 * run + b) % len(edges)], rng.integers(a0, a1))
            st.picks[:, :2].copy_(torch.from_numpy(pk))
            st.sirs.uniform_(-6, 6, generator=gen)
            st.snr.uniform_(10, 20, generator=gen)
            st.plan.run()
            snap = st.snap()
            torch.cuda.synchronize()
            c, n = check_snap(snap, nspk, nnoi, Ts, LEN, st.thr, "multi-group run %d" % run)
            total, near = total + c, near + n
            picks, starts = snap["picks"].cpu().numpy(), snap["starts"].cpu().numpy()
            seen |= {int(p) for p in picks[:, :2].reshape(-1)}
            for b in range(16):
                s = int(starts[b])
                crops = [x.full[:, s:s + LEN] for x in (nspk[picks[b, 0]], nspk[picks[b, 1]], nnoi[picks[b, 2]])]
                spk_f = torch.stack([fold_dev(crops[0]), fold_dev(crops[1])])
                mix, _ = _mix_dev(R, spk_f, fold_dev(crops[2])[None], st.sirs[b], st.snr[b])
                assert torch.equal(st.mix[b], mix), (run, b)
        print("multi-group draws: %d checked, %d near the threshold" % (total, near))
        assert set(edges) <= seen
        assert total >= 60 and near <= 2, (total, near)
        assert st.plan.is_graph()
        R.check_device_errors()
    finally:
        st.plan.close()
        sm.close()
        npool.close()


# ----------------------------------------------------------------------------------------- B. k_draw's warp edges
TRIES_SET = [1, 2, 31, 32, 33, 63, 64, 65, 101, 4095, 4096]


def beacon(rng, N, zoned):
    """A static 2-channel candidate: loud noise (about -10 dB) everywhere, and when `zoned` silent on [0, EDGE),
    [Z0, Z1) and [N - EDGE, N); a 64-tap RIR, so a crop at least 63 samples into a zone renders exact zeros."""
    x = so.synth_dry(rng, N) * np.float32(3.0)
    if zoned:
        x[:EDGE] = 0.0
        x[Z0:Z1] = 0.0
        x[N - EDGE:] = 0.0
    h = np.zeros((2, LB), np.float32)
    h[:, 0] = 1.0
    h[:, 1:] = rng.standard_normal((2, LB - 1)) * 0.05 * np.exp(-np.arange(1, LB) / 16.0)
    return Cand(x, h, None)


@pytest.fixture(scope="module")
def beacons():
    render, R = _R()
    rng = np.random.default_rng(305)
    # speakers 0 zoned short, 1 loud short, 2 zoned long, 3 loud long (the last the longest); noises long and shortest
    spk = [beacon(rng, NS, True), beacon(rng, NS, False), beacon(rng, NL, True), beacon(rng, NL, False)]
    noi = [beacon(rng, NL, False), beacon(rng, NN, False)]
    bw = types.SimpleNamespace(spk=spk, noi=noi)
    bw.ys = [host_stem(R, render, c)[0] for c in spk]
    bw.yn = [host_stem(R, render, c)[0] for c in noi]
    bw.T = [dr.level_table(y, True) for y in bw.ys]
    bw.full = {("spk", i): torch.from_numpy(y).cuda() for i, y in enumerate(bw.ys)}
    bw.full.update({("noi", i): torch.from_numpy(y).cuda() for i, y in enumerate(bw.yn)})
    bw.N = {("spk", i): c.N for i, c in enumerate(spk)}
    bw.N.update({("noi", i): c.N for i, c in enumerate(noi)})
    bw.sp = R.source_pool([c.src for c in spk], levels="mono")
    bw.np = R.source_pool([c.src for c in noi])
    yield bw
    bw.sp.close()
    bw.np.close()


# (readers, reader lane of speaker 0, 1, ..., the silent speaker, the shortest reader's lane or None: all long)


def combos():
    for tries in TRIES_SET:
        for t in sorted({t for t in TSTARS if t < tries} | {tries - 1}) + [None]:
            yield tries, t


def cases_of(layouts, seeds=(0,)):
    out = []
    for seed in seeds:
        for n, (tries, t) in enumerate(combos()):
            for j, lay in enumerate(layouts):
                out.append(Case(lay, tries, t, False, 1000 * seed + 17 * n + j))
                if tries > 37 and (t is None or t > 36) and seed == 0:
                    out.append(Case(lay, tries, t, True, 1000 * seed + 17 * n + j + 7))
    return out


class DrawPlan:
    """A plan of the cases' draws: one start and `used` element per draw, every reader a pooled slot of (2, WB) with
    the draw's start; NaN-filled outputs."""

    def __init__(self, R, render, bw, cases):
        self.cases = cases
        nd = len(cases)
        self.starts = torch.zeros(nd, dtype=torch.int32, device="cuda")
        self.used = torch.full((nd,), -7, dtype=torch.int32, device="cuda")
        self.u = torch.from_numpy(np.concatenate([c.u for c in cases])).cuda()
        pk = [c.bad_pick if (c.bad_pick is not None and j == 0) else i for c in cases for j, (_, i) in enumerate(c.lanes)]
        self.picks = torch.tensor(pk, dtype=torch.int32, device="cuda")
        self.out = torch.empty((len(pk), 2, WB), device="cuda")
        srcs, draws, off = [], [], 0
        self.slot0 = []
        for k, c in enumerate(cases):
            base = len(srcs)
            self.slot0.append(base)
            for j, (p, _) in enumerate(c.lanes):
                srcs.append(render.Pooled(bw.sp if p == "spk" else bw.np, self.picks[base + j], (self.starts[k], WB)))
            draws.append(render.CropDraw(self.starts[k], [base + lane for lane in c.speakers],
                                         self.u[off:off + c.tries], self.used[k]))
            off += c.tries
        self.plan = R.plan_device(srcs, [self.out[i] for i in range(len(srcs))], draws=draws)

    def run(self):
        self.out.fill_(NAN)
        self.starts.fill_(-1)
        self.plan.run()
        torch.cuda.synchronize()

    def check(self, bw, what):
        starts, used = self.starts.cpu().numpy(), self.used.cpu().numpy()
        for k, c in enumerate(self.cases):
            label = (what, k, c.layout, c.tries, c.tstar)
            got = (int(starts[k]), int(used[k]))
            assert got == (c.start, c.used), (label, got, (c.start, c.used))
            tabs = [bw.T[c.lanes[lane][1]] for lane in c.speakers]
            Nr = [bw.N[x] for x in c.lanes]
            D = [WB] * len(tabs)
            assert dr.draw(tabs, D, Nr, WB, c.u) == got, label
            assert dr.margins(tabs, D, Nr, WB, c.u) > 20.0, label        # every evaluated try far from -40 dB
            s = got[0]
            for j, x in enumerate(c.lanes):
                assert torch.equal(self.out[self.slot0[k] + j], bw.full[x][:, s:s + WB]), (label, j)

    def close(self):
        self.plan.close()


def test_draw_warp_edges(beacons):
    """Plans of 1, 3, 4 and 5 draws and then plans of 50 over the 16-reader layouts, and one plan of about 1000 draws
    over the small ones; every run is checked against the design and draw_reference."""
    render, R = _R()
    large = cases_of(LARGE)
    small = cases_of(SMALL, seeds=(0, 1))
    small = small[:997]                                          # 997 = 4 * 249 + 1: the last CTA holds one draw
    sizes = [1, 3, 4, 5]
    chunks, at = [], 0
    for n in sizes:
        chunks.append(large[at:at + n])
        at += n
    while at < len(large):
        chunks.append(large[at:at + 50])
        at += 50
    chunks.append(small)
    assert len(small) == 997 and {len(ch) for ch in chunks[:4]} == set(sizes)
    outcomes = set()
    _device_errors(R)
    for n, ch in enumerate(chunks):
        dp = DrawPlan(R, render, beacons, ch)
        try:
            dp.run()
            assert _device_errors(R) == 0, n
            dp.check(beacons, "plan %d of %d draws" % (n, len(ch)))
            assert dp.plan.is_graph()
        finally:
            dp.close()
        outcomes |= {(c.tries, c.tstar) for c in ch}
    assert outcomes == set(combos())
    print("warp edges: %d draws in %d plans" % (len(large) + len(small), len(chunks)))


def test_out_of_range_pick_draws_from_the_clamped_candidate(beacons):
    """A speaker whose pick (-5) is clamped to candidate 0, the zoned short one: M and the silence of the first 40
    tries come from that candidate, ss_device_errors reports bit 3 alone, and its crop is candidate 0's."""
    render, R = _R()
    case = Case((3, [0, 1], 0, 0), 101, 40, True, 99)
    assert case.lanes[0] == ("spk", 0) and case.M == NS - WB + 1
    case.bad_pick = -5
    _device_errors(R)
    dp = DrawPlan(R, render, beacons, [case])
    try:
        for run in range(2):
            dp.run()
            assert _device_errors(R) == 8, run
            dp.check(beacons, "clamped pick, run %d" % run)
    finally:
        dp.close()
    assert _device_errors(R) == 0


# ----------------------------------------------------------------------------------------- C. k_levels tile edges
TILE = 2048                    # samples of one k_levels tile (256 threads x 8)
TILE_NS = [1, 7, TILE - 1, TILE, TILE + 1, 2 * TILE - 1, 2 * TILE, 2 * TILE + 1, 3 * TILE - 1, 3 * TILE + 1,
           8 * TILE - 1, 8 * TILE + 1]


@pytest.mark.parametrize("C", [1, 3, 5, 8])
def test_level_tables_at_tile_edges(C):
    render, R = _R()
    rng = np.random.default_rng(400 + C)
    cands = []
    for N in TILE_NS + [5 * TILE + 3]:
        x = so.synth_dry(rng, N)
        if N == 5 * TILE + 3:
            x[500:9000] = 0.0                                    # zero terms over whole tiles 1 to 3: the carry alone
        h = np.zeros((C, 16), np.float32)
        h[:, 0] = 1.0
        h[:, 1:] = rng.standard_normal((C, 15)) * 0.3 * np.exp(-np.arange(1, 16) / 4.0)
        cands.append(Cand(x, h, None))
    ys = [host_stem(R, render, c)[0] for c in cands]
    assert np.abs(ys[-1][:, 600:8900]).max() < 1e-5 * np.abs(ys[-1]).max()
    worst = 0.0
    for levels in ("mono", "channels"):
        a = R.source_pool([c.src for c in cands], levels=levels)
        b = R.source_pool([c.src for c in cands], levels=levels)
        try:
            for i, (c, y) in enumerate(zip(cands, ys)):
                q = a.level_table(i)
                assert torch.equal(q, b.level_table(i)), (C, levels, c.N)
                r = table_error(q.cpu().numpy(), y, levels == "mono")
                assert r <= TABLE_TOL, (C, levels, c.N, r / TABLE_TOL)
                worst = max(worst, r)
        finally:
            a.close()
            b.close()
    print("C = %d: worst tile-edge table error %.3g x TABLE_TOL" % (C, worst / TABLE_TOL))
