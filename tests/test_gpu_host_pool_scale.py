"""Host pools (SS_BANK_HOST) at training scale against float64.  A slot of a host pool renders from what k_stage copied
into its staging area at that run (stage_set's dry samples and RIR rows, StageView), so a staging overrun, a wrong row
origin (h_row0) or a view given to the wrong slot gives plausible audio.  Every output here is checked (i) bit for bit
against the same plan over device pools of the same candidates, and (ii) sample by sample against float64
(render_reference.check_render; a pool with loudness gains scales the reference by its float32 gain; direct stems
against direct_path_rirs).  Outputs lie in NaN-filled buffers with sentinels on both sides (test_gpu_plan_scale.Out).
  A. staged crops on both blockings: grid, aligned (direct targets), mixed-K and static host pools with N % 4 in
     {1, 2, 3}, pure-delay RIRs and graded dry signals; starts 0 and N - len, the maximisers of stage_cap, both clamps of
     the read set and starts with ws % 4 in {1, 2, 3}, for windows of 64 000, 3 * 4096 + 5 and 3001 samples and fixed
     starts; the slots whose read sets fill the staging area run side by side;
  B. training scale: configs[1] speakers with direct targets (default budget and one chunk), P = 60 speakers with random
     cuts over 32 shared RIR sets with loudness gains, and K = 1..4 speakers in 48 slots; mixtures against
     mix_reference, draws against draw_reference on the pool's own tables;
  C. a plan that interleaves host-pool, device-pool, dry-picked and unpooled slots and a static source over every kernel
     variant (launches: the device-pool plan's plus one; one graph; a side stream), and a plan of 1056 host-pool slots;
  D. host-pool builds whose copy batches split stem groups (48 P = 60 speakers) and a candidate whose copy alone exceeds
     256 MiB: LUFS, gains and tables against the device-pool twin, render_host, the float64 BS.1770 oracle and the
     long-double prefix; a training plan with draws over the speaker pool.
No test holds more than 2 GB of pinned host memory in banks and pools (as counted by their host_nbytes)."""
import numpy as np
import pytest
import torch

from chunk_budget import DEFAULT_CHUNK_BYTES, chunk_budget  # noqa: F401  (fixture)
from oracle import sonicsim_oracle as so
from window_cases import stage_set_np
from draw_reference import TABLE_TOL, gappy_dry
from gpu_plumbing import _R, to
from mix_reference import Out
from pool_worlds import (A_LENS, STEM_BYTES, Pools, Probes, ScaleCand, _hold, _random_cuts, _training, a_aligned,
                         a_grid, a_mixed_k, a_static, align_up, b_configs1, copy_batches, d_giant, d_speakers,
                         host_alone, probe_starts, read_set, report as _report, stem_groups, table_error)
from window_cases import _choice

pytestmark = pytest.mark.gpu

RATE = 16000
B = 4096
TAPS = 40
ONE_CHUNK = 1 << 30


# ----------------------------------------------------------------------------------------- A. staged crops
A_POOLS = {"grid": (a_grid, False, "k_render<0,0>"), "aligned": (a_aligned, True, "k_render_fast"),
           "mixed-K": (a_mixed_k, False, "k_render<1,0>"), "static": (a_static, False, "k_render_fast static")}


@pytest.mark.parametrize("kind", list(A_POOLS))
def test_staged_crops_at_every_read_set_edge(kind):
    make, taps, variant = A_POOLS[kind]
    render, R = _R()
    rng = np.random.default_rng(600 + len(kind))
    cands = make(rng)
    assert {c.N % 4 for c in cands} >= ({1, 2, 3} if len(cands) >= 3 else {1, 2})
    pl = Pools(cands, taps=taps)
    assert pl.variant == variant, (kind, pl.variant)
    _hold(pl)
    k = 8
    n_min = min(c.N for c in cands)
    fixed = [n_min - wl for wl in A_LENS]
    pr = Probes(pl, A_LENS, k, fixed)
    sets = 2 if taps else 1
    try:
        R.check_device_errors()
        queues = []
        for wl in A_LENS:                      # the largest read sets first, so that the full areas run side by side
            q = [read_set(c, s, wl, sets) + (i, s) for i, c in enumerate(cands) for s in probe_starts(c, wl, rng)]
            q.sort(key=lambda t: -t[0])
            queues.append(q)
        # the staging area: the most rows and dry samples of any read set (the probes hold stage_cap's maximisers)
        cap = {wl: (max(t[1] for t in q), max(t[2] for t in q)) for wl, q in zip(A_LENS, queues)}
        runs = max(-(-len(q) // k) for q in queues)
        full_together = 0
        for r in range(runs):
            pk, st = [], []
            for wl, q in zip(A_LENS, queues):
                take = q[r * k:(r + 1) * k]
                while len(take) < k:                   # the rest: random picks and starts
                    i = int(rng.integers(0, len(cands)))
                    take.append((0, -1, -1, i, int(rng.integers(0, cands[i].N - wl + 1))))
                full_together = max(full_together, sum(t[1] == cap[wl][0] or t[2] == cap[wl][1] for t in take))
                pk += [t[3] for t in take] + [int(rng.integers(0, len(cands)))]
                st += [t[4] for t in take] + [0]
            pr.run(pk, st)
            pr.check("A %s" % variant, "%s run %d" % (kind, r))
        assert full_together >= 2, full_together                        # full staging areas side by side
        R.check_device_errors()
        print("\n%s: %d runs of %d slots; staging capacity reached by %d adjacent slots" %
              (kind, runs, len(pr.slots), full_together))
        _report("A")
    finally:
        pr.close()
        pl.close()


# ----------------------------------------------------------------------------------------- B. training scale


@pytest.mark.parametrize("budget", ["default", "one-chunk"])
def test_training_configs1_pool(budget, chunk_budget):
    R = chunk_budget(DEFAULT_CHUNK_BYTES if budget == "default" else ONE_CHUNK)
    rng = np.random.default_rng(701)
    spk, noi = b_configs1(rng)
    pools = {"spk": Pools(spk, taps=True, levels="mono"), "noi": Pools(noi)}
    _hold(*pools.values())
    try:
        _training(pools, [("spk", True), ("spk", True), ("noi", False)], "configs1 %s" % budget)
        _report("B configs1 %s" % budget)
    finally:
        for p in pools.values():
            p.close()
    assert R


def test_training_p60_pool_with_gains():
    """P = 60 with random cuts (some candidates on the grid) over 32 shared RIR sets, loudness targets; 2 speakers, a
    noise and a music per example."""
    rng = np.random.default_rng(702)
    N, P, C = 30 * RATE, 60, 6
    rirs = [so.synth_rirs(rng, P, C, 4096) for _ in range(32)]
    spk = [ScaleCand(gappy_dry(rng, N) if j % 3 == 0 else so.synth_dry(rng, N), rirs[j % 32],
                _random_cuts(rng, P, N, None if j % 4 else 60000))
           for j in range(40)]
    assert {_choice(c.b, N, P, 4096) for c in spk} == {0, 1}
    stat = [ScaleCand(so.synth_dry(rng, N - 1000 * j),
                 (rng.standard_normal((1, C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32), None)
            for j in range(16)]
    targets = [float(rng.uniform(-30, -16)) if j % 5 else None for j in range(len(spk))]
    pools = {"spk": Pools(spk, levels="mono", lufs=targets, share=[j % 32 for j in range(len(spk))]),
             "noi": Pools(stat[:8]), "mus": Pools(stat[8:])}
    _hold(*pools.values())
    try:
        assert np.array_equal(pools["spk"].pools[False].loudness, pools["spk"].pools[True].loudness, equal_nan=True)
        _training(pools, [("spk", False), ("spk", False), ("noi", False), ("mus", False)], "P=60 gains")
        _report("B P=60 gains")
    finally:
        for p in pools.values():
            p.close()


def test_training_mixed_k_pool():
    """32 configs[1]-shaped speakers with K = 1..4 in 48 slots (3 per scene)."""
    import bench
    rng = np.random.default_rng(703)
    items = bench.make_inputs(16, 0)
    Ls = (4096, 8192, 12288, 16384)
    spk = []
    for j, (x, h, b) in enumerate(items):
        L = Ls[j % 4]
        hh = h if L == 4096 else so.synth_rirs(rng, h.shape[0], h.shape[1], L)
        spk.append(ScaleCand(gappy_dry(rng, len(x)) if j % 2 else x, hh, b))
    pools = {"spk": Pools(spk, levels="mono")}
    _hold(*pools.values())
    try:
        _training(pools, [("spk", False)] * 3, "mixed-K")
        _report("B mixed-K")
    finally:
        for p in pools.values():
            p.close()


# ----------------------------------------------------------------------------------------- C. mixed plans
def test_mixed_plan_of_host_device_dry_and_unpooled_slots():
    """Caller order interleaves host-pool slots (grid and aligned), device-pool slots, dry-picked device-pool slots,
    unpooled banked moving sources (fast, long) and a static source; arrange_chunks regroups them by kernel variant."""
    render, R = _R()
    rng = np.random.default_rng(801)
    grid, aligned = Pools(a_grid(rng)), Pools(a_aligned(rng), taps=True)
    dev = Pools(a_aligned(rng))
    longs = [ScaleCand(so.synth_dry(rng, 40000 + 3 * j), so.synth_rirs(rng, 3, 2, 9000),
                  np.array([0, 15000 + j, 40000 + 3 * j], np.int32)) for j in range(2)]
    static = ScaleCand(so.synth_dry(rng, 50001), so.synth_rirs(rng, 1, 2, 2048), None)
    _hold(grid, aligned, dev)
    dry = [so.synth_dry(rng, 140000) for _ in range(3)]
    dpool = R.dry_pool([to(x) for x in dry])
    banks = [R.rir_bank(to(c.h)) for c in longs] + [R.rir_bank(to(static.h[0]))]
    wl = 20001
    kinds = ["host grid", "device", "unpooled long", "host aligned", "dry", "static", "host grid", "unpooled long",
             "device", "host aligned", "dry", "host grid"]
    n = len(kinds)
    picks = torch.zeros(n, dtype=torch.int32, device="cuda")
    dpicks = torch.zeros(n, dtype=torch.int32, device="cuda")
    starts = torch.zeros(n, dtype=torch.int32, device="cuda")

    def sources(host):
        srcs, unp = [], 0
        for j, k in enumerate(kinds):
            w = (starts[j], wl)
            if k == "host grid":
                srcs.append(render.Pooled(grid.pools[host], picks[j], w))
            elif k == "host aligned":
                srcs.append(render.Pooled(aligned.pools[host], picks[j], w, TAPS))
            elif k == "device":
                srcs.append(render.Pooled(dev.pools[False], picks[j], w))
            elif k == "dry":
                srcs.append(render.Pooled(dev.pools[False], picks[j], w, dry=render.DryPick(dpool, dpicks[j])))
            elif k == "unpooled long":
                c = longs[unp]
                srcs.append(render.MovingSource(to(c.x), banks[unp], to(c.b), c.b, window=w))
                unp += 1
            else:
                srcs.append(render.StaticSource(to(static.x), banks[2], window=w))
        return srcs

    C = [3 if k == "host grid" else 2 for k in kinds]
    outs = {h: [Out(c, wl) for c in C] for h in (False, True)}
    douts = {h: [Out(2, wl) if k == "host aligned" else None for k in kinds] for h in (False, True)}
    plans = {h: R.plan_device(sources(h), [o.view() for o in outs[h]],
                              direct_outs=[None if o is None else o.view() for o in douts[h]]) for h in (False, True)}
    try:
        R.check_device_errors()
        counts = {}
        for run in range(4):
            pk, dp, st = [], [], []
            for j, k in enumerate(kinds):
                if k.startswith("host"):
                    cs = (grid if "grid" in k else aligned).cands
                elif k in ("device", "dry"):
                    cs = dev.cands
                else:
                    cs = longs if "long" in k else [static]
                i = int(rng.integers(0, len(cs))) if k != "unpooled long" else kinds[:j].count(k)
                N = cs[i].N if k != "static" else static.N
                pk.append(i if k != "static" else 0)
                dp.append(int(rng.integers(0, len(dry))))
                st.append((0, N - wl, int(rng.integers(0, N - wl + 1)), N - wl - 2 * B + 1)[(run + j) % 4])
            picks.copy_(torch.tensor(pk, dtype=torch.int32))
            dpicks.copy_(torch.tensor(dp, dtype=torch.int32))
            starts.copy_(torch.tensor(st, dtype=torch.int32))
            for h in (False, True):
                for o in outs[h] + [x for x in douts[h] if x is not None]:
                    o.reset()
                R.reset_stats()
                plans[h].run()
                counts[h] = R.launch_count()
            torch.cuda.synchronize()
            if run > 0:
                assert counts[True] == counts[False] + 1, counts
            for j, k in enumerate(kinds):
                y = outs[True][j].get()
                assert np.array_equal(y, outs[False][j].get()), (run, j, k)
                label = "mixed plan run %d slot %d (%s)" % (run, j, k)
                if k.startswith("host"):
                    c = (grid if "grid" in k else aligned).cands[pk[j]]
                elif k == "device":
                    c = dev.cands[pk[j]]
                elif k == "dry":
                    d = dev.cands[pk[j]]
                    c = ScaleCand(dry[dp[j]][:d.N], d.h, d.b)
                elif k == "unpooled long":
                    c = longs[pk[j]]
                else:
                    c = static
                c.check(y, st[j], wl, key="C mixed %s" % k, label=label)
                if douts[True][j] is not None:
                    yd = douts[True][j].get()
                    assert np.array_equal(yd, douts[False][j].get()), (run, j, k)
                    c.check(yd, st[j], wl, direct=True, key="C mixed %s" % k, label=label + " direct")
        for p in plans.values():
            assert p.is_graph()
        # a side stream, behind queued work
        ref = [o.get().copy() for o in outs[True]]
        for o in outs[True]:
            o.reset()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            torch.cuda._sleep(int(2e7))
            plans[True].run(s.cuda_stream)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        for j, o in enumerate(outs[True]):
            assert np.array_equal(o.get(), ref[j]), ("side stream", j)
        R.check_device_errors()
        _report("C mixed")
    finally:
        for p in plans.values():
            p.close()
        for k in banks:
            k.close()
        dpool.close()
        for p in (grid, aligned, dev):
            p.close()


def stage_bytes(cands, wl, sets):
    """stage_bytes of ss_kernels.cu: the view, sets * rows_cap rows and nx_cap dry floats, each 256-aligned, with the
    capacity (stage_cap) the largest read set over every start of every candidate."""
    rows = nx = 0
    for c in cands:
        xa, xb, _, r = stage_set_np(c.N, c.P, c.C, c.K, c.b, np.arange(c.N - wl + 1), wl)
        rows, nx = max(rows, int(r.max())), max(nx, int((xb - xa).max()) + 8)
    return align_up(56, 256) + align_up(sets * rows * B * 8, 256) + align_up(4 * nx, 256)


def test_many_staged_slots():
    """1056 host-pool slots with 1500-sample windows over small candidates: a k_stage grid of 1056 rows and several
    chunks under the default budget."""
    render, R = _R()
    rng = np.random.default_rng(802)
    cands = []
    for j in range(6):
        N, P = 20001 + 1001 * j, 3 + j % 3
        cands.append(ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 1, 2000), _random_cuts(rng, P, N)))
    pl = Pools(cands)
    _hold(pl)
    n, wl = 1056, 1500
    pr = Probes(pl, [wl], n - 1, [123])
    try:
        for run in range(2):
            pk = rng.integers(0, len(cands), n)
            st = [int(rng.integers(0, cands[p].N - wl + 1)) for p in pk]
            pr.run(pk, st)
            # every slot in the first run (so the first and last staged slots, whatever order arrange_chunks gives
            # them), the first, last and 40 others in the second
            sample = range(n) if run == 0 else sorted({0, n - 1} | set(rng.choice(n, 40, replace=False).tolist()))
            for j in sample:
                c = cands[pr.pk[j]]
                c.check(pr.outs[True][j].get(), pr.st[j], wl, key="C many", label="many run %d slot %d" % (run, j))
        launches = pr.launches
        chunks = launches[False] / 3                     # k_blocks, k_prepare and the render per chunk
        print("\nmany slots: %d host-pool slots, %g chunks, launches per run %s (device, host pools), %d bytes of "
              "staging (restated stage_bytes)" % (n, chunks, launches, n * stage_bytes(cands, wl, 1)))
        assert launches[True] == launches[False] + 1 and chunks == int(chunks) and chunks > 1, launches
        R.check_device_errors()
        _report("C many")
    finally:
        pr.close()
        pl.close()


# ----------------------------------------------------------------------------------------- D. builds across batches


@pytest.mark.parametrize("kind", ["speakers", "giant"])
def test_host_builds_across_copy_batches(kind):
    render, R = _R()
    rng = np.random.default_rng(901 if kind == "speakers" else 902)
    cands = d_speakers(rng) if kind == "speakers" else d_giant(rng)
    C = cands[0].C
    first, _ = stem_groups(C, [c.N for c in cands])
    batches, cap = copy_batches(C, cands, first)
    inside = [s for s in batches if s not in first]
    print("\n%s: stem groups %s, copy batches %s, copy buffer %d bytes" % (kind, first, batches, cap))
    if kind == "speakers":
        assert inside, (first, batches)                   # a batch boundary strictly inside a stem group
        unmeasured = {inside[0], first[1], first[1] - 1}
        silent = {inside[0] - 1}
    else:
        assert cap > STEM_BYTES and 2 in batches and 3 in batches, (batches, cap)
        unmeasured, silent = {1}, {3}                      # on each side of the giant
    for j in silent:
        cands[j].x[:] = 0.0
    trng = np.random.default_rng(903)
    targets = [None if j in unmeasured else float(trng.uniform(-30, -14)) for j in range(len(cands))]
    refs = [host_alone(R, render, c, t) for c, t in zip(cands, targets)]
    oracle = [None if t is None or j in silent else
              so.bs1770_integrated_loudness(host_alone(R, render, c, None)[0].T.astype(np.float64), RATE, 0.4,
                                            up_to_8_channels=True) for j, (c, t) in enumerate(zip(cands, targets))]
    worst_tab = worst_db = 0.0
    for levels in ("mono", "channels"):
        pl = Pools(cands, levels=levels, lufs=targets)
        _hold(pl)
        try:
            Ld, Lh = pl.pools[False].loudness, pl.pools[True].loudness
            assert Ld.tobytes() == Lh.tobytes(), (kind, levels)
            for i, (c, t) in enumerate(zip(cands, targets)):
                what = (kind, levels, i)
                q = pl.pools[True].level_table(i)
                assert torch.equal(q, pl.pools[False].level_table(i)), what
                y, lo = refs[i]
                if t is None:
                    assert np.isnan(Lh[i]).all(), what
                else:
                    assert (Lh[i, 0], Lh[i, 1]) == lo, (what, Lh[i], lo)
                    if i in silent:
                        assert np.isneginf(Lh[i, 0]), what
                    else:
                        d = abs(Lh[i, 0] - oracle[i])
                        assert d < 1e-6, (what, Lh[i, 0], oracle[i])
                        worst_db = max(worst_db, d)
                r = table_error(q.cpu().numpy(), y, levels == "mono")
                assert r <= TABLE_TOL, (what, r / TABLE_TOL)
                worst_tab = max(worst_tab, r)
            if kind == "speakers" and levels == "mono":
                _training({"spk": pl}, [("spk", False)] * 3, "D speakers", runs=2, min_draws=20)
        finally:
            pl.close()
    print("%s: worst table error %.3g x TABLE_TOL, worst loudness vs the oracle %.3g dB" %
          (kind, worst_tab / TABLE_TOL, worst_db))
