"""16-bit dry pools (Renderer.dry_pool(..., dtype="int16"), ss_dry_pool_create_i16) at training scale against float64.
A 16-bit pool shares k_levels, draw_silent_sums and the staging sizes with a float pool, so a fault there gives the
same wrong bits in both; what it adds is its own sample expansion (i16_sample), its sparse tables (k_level_sample,
sparse_level) and its arena offsets.  Sample k stands for k / 32768, exactly a float32, so the float64 reference
(render_reference.render_f64 of those values, through ScaleCand.check on a thread pool) sees exactly what the device
sees.  Every plan runs twice, over the 16-bit pool and over a float32 pool of the same values, and the two must give the
same bits; every stem must also pass the float64 check, and every table must equal the long-double prefix of the
float32 squares exactly (==: the squares of 16-bit samples are multiples of 2^-30, DESIGN f13).  Outputs lie in
NaN-filled buffers with sentinels on both sides (mix_reference.Out).
  A. full-scale signals - runs of -32768 and of 32767, alternating full scale, isolated full-scale samples at residues
     0, 1, 62, 63 and 64 of the level stride, lengths with N % 64 in {0, 1, 63} and N % 4 in {1, 2, 3} - through the
     grid, aligned (direct targets), mixed-K and static pools, device and host source pools x device and host 16-bit
     pools; their level tables and raw sparse tables;
  B. a plan of 1040 slots over device source pools - 16-bit dry picks (staged only because their pool is 16-bit), float
     dry picks and plain slots - under the default and a small chunk budget, and a second plan over the same 16-bit pool
     run in turn with it;
  C. draws: the warp-edge beacon cases of pool_worlds (Case: every tries count and kept try, speakers at every reader
     lane) on the int16 grid, every draw mixing 16-bit and float speakers; and designed crops that begin and end at
     every residue of the level stride, whose verdict hinges on one full-scale square at a stride-block edge, so that
     sparse_level sums 0 to 63 squares at either end - starts and `used` against the designed outcomes and
     draw_reference on the exact tables;
  D. a device 16-bit pool of 257 signals of about 2^23 samples whose arena passes 2^32 bytes, with signals straddling
     the 2^31 and 2^32 byte offsets: nbytes, tables, stems and draws of slots that pick them; a host pool of the same
     kind under 2 GB; the pool's own signal addresses give the layout, and its table build runs in several expansion
     batches.
Not here: one training plan that combines tap-form speakers, 16-bit dry picks with pair gains and dereverberation
targets, float host noise picks and mixtures across chunks.  Each of those is checked against float64 above, in
test_gpu_taps_pool_scale or in test_gpu_plan_target; their combination in one plan is left to a test of its own."""
import ctypes

import numpy as np
import pytest
import torch

import draw_reference as dr
from chunk_budget import DEFAULT_CHUNK_BYTES, chunk_budget  # noqa: F401  (fixture)
from gpu_plumbing import _R, _device_errors, pmap, to
from mix_reference import Out
from oracle import sonicsim_oracle as so
from pool_worlds import (B, LARGE, NAN, NL, NN, NS, PINNED_MAX, SMALL, STEM_BYTES, TAPS, Cand, DevPool, DryDrawPlan,
                         Pools, ScaleCand, a_aligned, a_grid, a_mixed_k, a_static, align_up, d_cases, d_combos,
                         dry_beacon, probe_starts, report, traj_beacon)

pytestmark = pytest.mark.gpu

STRIDE = 64                                  # kLevelStride
FULL = (-32768, 32767)


def values(k):
    return k.astype(np.float32) / np.float32(32768)


def exact_table(k):
    """The level table of 16-bit samples k: the long-double prefix of the float32 squares of k / 32768 (exact: every
    square is a multiple of 2^-30 and the sums stay below 2^23), as float64."""
    return dr.level_table(values(k)[None], True, np.longdouble).astype(np.float64)


def sparse_of(ref, N):
    return ref[np.minimum(np.arange(-(-N // STRIDE) + 1) * STRIDE, N)]


def check_tables(pool, i, k, what):
    """level_table(i) and the raw sparse table against the exact prefix, with ==."""
    _, R = _R()
    ref = exact_table(k)
    q = pool.level_table(i).cpu().numpy()
    assert q.shape == ref.shape and np.array_equal(q, ref), (what, i, len(k))
    raw = pool._read(R.lib.ss_dry_pool_level_table(pool._h, i), -(-len(k) // STRIDE) + 1, "<f8", ctypes.c_double)
    assert np.array_equal(raw, sparse_of(ref, len(k))), (what, "sparse", i)


def full_scale_i16(rng, N, j):
    """Speech-like noise up to full scale with runs of -32768 and of 32767, alternating full scale, and isolated
    full-scale samples at residues 0, 1, 62, 63 and 64 of the level stride amid silence."""
    v = so.synth_dry(rng, N).astype(np.float64)
    k = np.clip(np.round(v / np.abs(v).max() * 32768.0 * 1.2), -32768, 32767).astype(np.int16)   # clipped peaks
    for at in range(4000 + 1000 * j, N - 3000, 23000):
        n = int(rng.integers(40, 600))
        k[at:at + n] = FULL[(at // 23000) % 2]                      # runs of -32768 and of 32767
        k[at + n:at + n + 333] = np.where(np.arange(333) % 2, 32767, -32768)     # alternating
        z = at + n + 333 + (-(at + n + 333)) % STRIDE + STRIDE      # a silent stretch on a stride boundary ...
        k[z:z + 3 * STRIDE] = 0
        for r in (0, 1, 62, 63, 64):                                # ... with isolated full-scale samples
            k[z + r] = FULL[r % 2]
    return k


def lengths_for(n_max):
    """Lengths of at least n_max with N % 64 in {0, 1, 63} and N % 4 in {1, 2, 3}."""
    m = -(-n_max // STRIDE) * STRIDE
    return [m, m + 1, m + 63, m + 66, m + 64 + 3]


def twin(R, ks, resident, i16_resident, levels=False):
    """The float32 pool (host when the source pool is) and the 16-bit pool of the same values."""
    fl = [values(k) for k in ks]
    fp = R.dry_pool(fl, levels=levels, host=True) if resident == "host" else R.dry_pool([to(x) for x in fl],
                                                                                       levels=levels)
    ip = R.dry_pool(ks, levels=levels, host=i16_resident == "host", dtype="int16")
    assert ip.dtype == "int16" and ip.level_stride == STRIDE and ip.sizes == fp.sizes
    return fp, ip


def hold(*pools):
    """The pinned host bytes of the source pools (Pools.pinned) and dry pools (host_nbytes) a test holds, printed and
    kept under 2 GB."""
    total = sum(p.pinned if isinstance(p, Pools) else p.host_nbytes for p in pools)
    print("\npinned host memory of the banks and pools held (host_nbytes): %.1f MB" % (total / 1e6))
    assert total <= PINNED_MAX, total


def f64(jobs):
    pmap(lambda t: t[0].check(t[1], t[2], t[3], direct=t[4], key=t[5], label=t[6]), jobs)


class I16Slots:
    """Dry-picked slots of one source pool over one dry pool, (picks, dry picks, starts) in device memory."""

    def __init__(self, pool, dp, C, lens, k, taps=0):
        render, R = _R()
        self.slots = [wl for wl in lens for _ in range(k)]
        n = len(self.slots)
        self.vals = torch.zeros((3, n), dtype=torch.int32, device="cuda")
        self.outs = [Out(C, wl) for wl in self.slots]
        self.douts = [Out(C, wl) for wl in self.slots] if taps else []
        srcs = [render.Pooled(pool, self.vals[0, j], (self.vals[2, j], wl), taps, render.DryPick(dp, self.vals[1, j]))
                for j, wl in enumerate(self.slots)]
        self.plan = R.plan_device(srcs, [o.view() for o in self.outs],
                                  direct_outs=[o.view() for o in self.douts] if taps else None)

    def run(self, v):
        for o in self.outs + self.douts:
            o.reset()
        self.vals.copy_(to(v))
        self.plan.run()
        torch.cuda.synchronize()
        return [o.get().copy() for o in self.outs + self.douts]

    def close(self):
        self.plan.close()


# ----------------------------------------------------------------------------------------- A. full-scale signals
A_POOLS = {"grid": a_grid, "aligned": a_aligned, "mixed-K": a_mixed_k, "static": a_static}
A_LENS = [3001, 3 * B + 5, 64000]


@pytest.mark.parametrize("kind", list(A_POOLS))
def test_full_scale_signals(kind):
    make = A_POOLS[kind]
    R = _R()[1]
    rng = np.random.default_rng(3100 + len(kind))
    cands = make(rng)
    taps = kind == "aligned"
    pl = Pools(cands, taps=taps)
    n_max = max(c.N for c in cands)
    ks = [full_scale_i16(rng, n, j) for j, n in enumerate(lengths_for(n_max))]
    assert {len(k) % 64 for k in ks} >= {0, 1, 63} and {len(k) % 4 for k in ks} >= {1, 2, 3}
    assert all((k == -32768).sum() > 200 and (k == 32767).sum() > 200 for k in ks)
    xs = [values(k) for k in ks]
    k_slots, C = 4, cands[0].C
    arms = {}
    try:
        for res in ("device", "host"):
            for i16_res in ("device", "host"):
                fp, ip = twin(R, ks, res, i16_res, levels=True)
                pool = pl.pools[res == "host"]
                hold(pl, fp, ip)
                arms[res, i16_res] = (fp, ip, I16Slots(pool, fp, C, A_LENS, k_slots, TAPS if taps else 0),
                                      I16Slots(pool, ip, C, A_LENS, k_slots, TAPS if taps else 0))
                for i, k in enumerate(ks):
                    check_tables(ip, i, k, (kind, res, i16_res))
        queues = [[(i, s) for i, c in enumerate(cands) for s in probe_starts(c, wl, rng)] for wl in A_LENS]
        runs = max(-(-len(q) // k_slots) for q in queues)
        n = len(A_LENS) * k_slots
        full_hits = 0
        for r in range(runs):
            v = np.zeros((3, n), np.int32)
            for w, (wl, q) in enumerate(zip(A_LENS, queues)):
                for j in range(k_slots):
                    i, s = q[r * k_slots + j] if r * k_slots + j < len(q) else (0, 0)
                    v[:, w * k_slots + j] = i, (r + j + w) % len(ks), s
            ref = None
            for key, (fp, ip, fs, is_) in arms.items():
                a, b = fs.run(v), is_.run(v)
                for j, (x, y) in enumerate(zip(a, b)):
                    assert np.array_equal(x, y), (kind, key, r, j)
                if ref is None:
                    ref = b
                else:
                    for j, (x, y) in enumerate(zip(ref, b)):
                        assert np.array_equal(x, y), (kind, key, "against the device arms", r, j)
            jobs = []
            for j, wl in enumerate(arms["device", "device"][3].slots):
                i, d, s = (int(t) for t in v[:, j])
                c = cands[i]
                ref_c = ScaleCand(xs[d][:c.N], c.h, c.b)
                full_hits += int(np.isin(ks[d][max(0, s - c.L):s + wl], FULL).sum())
                what = "%s run %d slot %d cand %d dry %d start %d len %d" % (kind, r, j, i, d, s, wl)
                jobs.append((ref_c, ref[j], s, wl, False, "A 16-bit %s" % kind, what))
                if taps:
                    jobs.append((ref_c, ref[n + j], s, wl, True, "A 16-bit %s" % kind, what + " direct"))
            f64(jobs)
        assert full_hits > 1000, full_hits                 # full-scale samples rendered into the checked crops
        R.check_device_errors()
        print("\n%s: %d runs of %d slots over 4 residency pairs; %d full-scale samples read by checked crops" %
              (kind, runs, n, full_hits))
        report("A 16-bit")
    finally:
        for fp, ip, fs, is_ in arms.values():
            fs.close()
            is_.close()
            fp.close()
            ip.close()
        pl.close()


# ----------------------------------------------------------------------------------------- B. plan scale
def b_pools(rng):
    aligned = [ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, B), np.round(np.linspace(0, N, P)).astype(np.int32))
               for N, P in ((20001, 3), (24002, 4), (28003, 3))]
    longs = [ScaleCand(so.synth_dry(rng, N), so.synth_rirs(rng, 3, 2, L), np.round(np.linspace(0, N, 3)).astype(np.int32))
             for N, L in ((21001, 9000), (26002, 5000))]
    return {"aligned": Pools(aligned, host_only=False), "long": Pools(longs)}


B_KINDS = ["i16 aligned", "float aligned", "plain long", "i16 long", "plain aligned", "float long", "i16 aligned",
           "i16 long"]
B_WL = 1500


class BigPlan:
    """n slots cycling B_KINDS over the device arms of the pools; `arm` "i16" or "float" gives the 16-bit slots their
    16-bit pool or the float twin."""

    def __init__(self, pools, ip, fp, fl2, n, arm):
        render, R = _R()
        self.kinds = [B_KINDS[j % len(B_KINDS)] for j in range(n)]
        self.vals = torch.zeros((3, n), dtype=torch.int32, device="cuda")
        srcs = []
        for j, k in enumerate(self.kinds):
            how, key = k.split()
            dry = None
            if how == "i16":
                dry = render.DryPick(ip if arm == "i16" else fp, self.vals[1, j])
            elif how == "float":
                dry = render.DryPick(fl2, self.vals[1, j])
            srcs.append(render.Pooled(pools[key].pools[False], self.vals[0, j], (self.vals[2, j], B_WL), 0, dry))
        self.outs = [Out(2, B_WL) for _ in range(n)]
        self.plan = R.plan_device(srcs, [o.view() for o in self.outs])

    def run(self, v):
        for o in self.outs:
            o.reset()
        self.vals.copy_(to(v))
        self.plan.run()
        torch.cuda.synchronize()
        return [o.get().copy() for o in self.outs]

    def close(self):
        self.plan.close()


def test_plan_of_16_bit_float_and_plain_slots(chunk_budget):
    R = _R()[1]
    rng = np.random.default_rng(3201)
    pools = b_pools(rng)
    n_max = max(c.N for p in pools.values() for c in p.cands)
    ks = [full_scale_i16(rng, n, j) for j, n in enumerate(lengths_for(n_max) + [n_max + 7, n_max + 130])]
    fp, ip = twin(R, ks, "device", "device")
    f2 = [so.synth_dry(rng, n_max + 9 * j) for j in range(4)]
    fl2 = R.dry_pool([to(x) for x in f2])
    hold(*pools.values(), fp, ip, fl2)
    n = 1040
    v = np.zeros((3, n), np.int32)
    kinds = [B_KINDS[j % len(B_KINDS)] for j in range(n)]
    for j, k in enumerate(kinds):
        p = pools[k.split()[1]]
        i = int(rng.integers(0, len(p.cands)))
        nd = len(ks) if k.startswith("i16") else len(f2)
        v[:, j] = i, int(rng.integers(0, nd)), int(rng.integers(0, p.cands[i].N - B_WL + 1))
    plans, counts, ref = [], {}, None
    try:
        for budget in (DEFAULT_CHUNK_BYTES, 2 << 20):
            chunk_budget(budget)
            a, b = BigPlan(pools, ip, fp, fl2, n, "i16"), BigPlan(pools, ip, fp, fl2, n, "float")
            plans += [a, b]
            R.reset_stats()
            ya = a.run(v)
            counts[budget] = R.launch_count()
            R.reset_stats()
            yb = b.run(v)
            R.check_device_errors()
            for j in range(n):
                assert np.array_equal(ya[j], yb[j]), (budget, j, kinds[j])
            if ref is None:
                jobs = []
                for j, k in enumerate(kinds):
                    how, key = k.split()
                    i, d, s = (int(t) for t in v[:, j])
                    c = pools[key].cands[i]
                    x = values(ks[d])[:c.N] if how == "i16" else f2[d][:c.N] if how == "float" else c.x
                    jobs.append((ScaleCand(x, c.h, c.b), ya[j], s, B_WL, False, "B %s" % k.split()[1],
                                 "plan slot %d (%s) cand %d dry %d start %d" % (j, k, i, d, s)))
                f64(jobs)
                ref = ya
            else:
                for j in range(n):
                    assert np.array_equal(ya[j], ref[j]), ("small budget", j)
        print("\n1040 slots: launches per run %s (default, 2 MB budget)" % list(counts.values()))
        assert counts[2 << 20] > counts[DEFAULT_CHUNK_BYTES] + 30, counts
        # a second plan over the same 16-bit pool, in turn with the first
        small = I16Slots(pools["aligned"].pools[False], ip, 2, [B_WL, 5000], 4)
        plans.append(small)
        v2 = np.zeros((3, len(small.slots)), np.int32)
        for j, wl in enumerate(small.slots):
            v2[:, j] = j % 3, (5 - j) % len(ks), (97 * j) % (pools["aligned"].cands[j % 3].N - wl + 1)
        s1 = plans[-3].run(v)
        s2 = small.run(v2)
        s3 = plans[-3].run(v)
        jobs = []
        for j, wl in enumerate(small.slots):
            i, d, s = (int(t) for t in v2[:, j])
            c = pools["aligned"].cands[i]
            jobs.append((ScaleCand(values(ks[d])[:c.N], c.h, c.b), s2[j], s, wl, False, "B second plan",
                         "second plan slot %d" % j))
        f64(jobs)
        for s in (s1, s3):
            for j in range(n):
                assert np.array_equal(s[j], ref[j]), ("in turn", j)
        R.check_device_errors()
        report("B")
    finally:
        for p in plans:
            p.close()
        for p in (fp, ip, fl2):
            p.close()
        for p in pools.values():
            p.close()


# ----------------------------------------------------------------------------------------- C. draws
def quantise(x):
    return np.clip(np.round(np.asarray(x, np.float64) * 32768.0), -32768, 32767).astype(np.int16)


@pytest.fixture(scope="module")
def i16_beacons():
    """The dry beacons of test_gpu_dry_pool_scale D on the int16 grid (their loud stretches clip at full scale, their
    zones stay exactly 0), as a float pool (bw.dp) and a 16-bit pool (bw.dp16) of the same values: Case's designed
    starts and outcomes hold unchanged.  Tables of the reference: the long-double prefix of the signals' squares and of
    the plain candidates' whole stems."""
    R = _R()[1]
    rng = np.random.default_rng(3501)
    tp = DevPool([traj_beacon(rng, NS), traj_beacon(rng, NL)], levels="mono")
    npl = DevPool([traj_beacon(rng, NL), traj_beacon(rng, NN)])
    ks = [quantise(dry_beacon(rng, NL, z)) for z in (NS, 0, NL, 0)]
    assert all((k == -32768).sum() > 1000 for k in ks)
    dry_d = [to(values(k)) for k in ks]
    bw = type("Beacons", (), {})()
    bw.tp, bw.np = tp, npl
    bw.dp = R.dry_pool(dry_d, levels=True)
    bw.dp16 = R.dry_pool(ks, levels=True, dtype="int16")
    for i, k in enumerate(ks):
        check_tables(bw.dp16, i, k, "beacons")
    bw.Td = [exact_table(k) for k in ks]
    full = {}
    for i in range(4):                                         # whole stems: dry-picked, plain, noise
        c = 0 if i < 2 else 1
        full[("dry", i)] = torch.from_numpy(tp.ref(c, dry_d[i], 0, tp.cands[c].N)[0]).cuda()
    for t in range(2):
        full[("plain", t)] = torch.from_numpy(tp.ref(t, None, 0, tp.cands[t].N)[0]).cuda()
        full[("noi", t)] = torch.from_numpy(npl.ref(t, None, 0, npl.cands[t].N)[0]).cuda()
    bw.full = full
    bw.Tp = [dr.level_table(full[("plain", t)].cpu().numpy(), True, np.longdouble).astype(np.float64) for t in range(2)]
    yield bw
    for p in (tp, npl, bw.dp, bw.dp16):
        p.close()


def test_draw_warp_edges_with_16_bit_speakers(i16_beacons):
    """k_draw<true>'s warp edges: the designed cases of every tries count and kept try, speakers at every reader lane,
    every other dry-picked speaker (alternating by draw and lane) a 16-bit pick and the rest float picks."""
    R = _R()[1]
    bw = i16_beacons
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
    _device_errors(R)
    outcomes, worst, n16, hi16, mixed = set(), np.inf, 0, 0, 0
    for n, ch in enumerate(chunks):
        dp = DryDrawPlan(bw, ch, dp16=bw.dp16)
        try:
            dp.run()
            assert _device_errors(R) == 0, n
            worst = min(worst, dp.check(bw, "plan %d of %d draws" % (n, len(ch))))
            assert dp.plan.is_graph()
            n16 += len(dp.lanes16)
            hi16 += sum(1 for k, j in dp.lanes16 if j >= 8 and j in ch[k].speakers)
            kinds = {}
            for k, c in enumerate(ch):
                for j in c.speakers:
                    if dp.what[k][j][0] == "dry":
                        kinds.setdefault(k, set()).add((k, j) in dp.lanes16)
            mixed += sum(1 for v in kinds.values() if v == {True, False})
        finally:
            dp.close()
        outcomes |= {(c.tries, c.tstar) for c in ch}
    assert outcomes == set(d_combos())
    assert hi16 >= 50 and mixed >= 100, (hi16, mixed)        # 16-bit speakers at lanes 8 to 15; mixed draws
    print("\n16-bit warp edges: %d draws in %d plans, least margin %.1f dB, %d 16-bit speaker picks (%d at lanes >= "
          "8), %d draws with 16-bit and float speakers" % (len(large) + len(small), len(chunks), worst, n16, hi16, mixed))


RW = 1024                        # crop of the residue draws: one full-scale sample in it is -30.1 dB, none is silent
SPAN = 3 * RW                    # samples of the signal per designed crop (a multiple of the stride)
RES_KINDS = {"between": False,          # full-scale samples just before and just after the crop
             "first": True,             # one at the crop's first sample
             "last": True,              # one at its last
             "block head": False,       # one at the head of the stride block the crop starts in (outside it)
             "end block head": True}    # one at the head of the block the crop ends in (inside it)


def residue_signal():
    """A 16-bit signal silent but for single full-scale samples (-32768, whose square is exactly 1) placed around one
    designed crop [s, s + RW) per (residue r of s, kind), and a loud tail.  s and s + RW both have residue r, so
    sparse_level sums 0 to 63 squares at either end; returns (samples, [(s, r, kind, loud)], start of the tail)."""
    designs = [(r, kind) for r in range(STRIDE) for kind in RES_KINDS]
    tail = len(designs) * SPAN
    k = np.zeros(tail + 2 * RW, np.int16)
    k[tail:] = np.where(np.arange(2 * RW) % 2, 32767, -32768)
    out = []
    for n, (r, kind) in enumerate(designs):
        s = n * SPAN + RW + r
        e = s + RW
        pos = {"between": [s - 1, e], "first": [s], "last": [e - 1], "block head": [s - r if r else s - STRIDE],
               "end block head": [e - r if r else e - STRIDE]}[kind]
        for q in pos:
            k[q] = -32768
        out.append((s, r, kind, RES_KINDS[kind]))
    return k, out, tail


def test_draws_at_every_residue_of_the_stride():
    """Each draw's first try is a designed crop whose level hinges on one square at a stride-block edge (the Q[s] of a
    16-bit speaker is its sparse table's entry plus the r squares in front of s), its second try the loud tail: kept
    try 1 for a loud crop, 2 for a silent one.  The residue speaker is a 16-bit pick in one plan and a float pick of the
    same values in the other, at lane 0 or 1 next to a loud float speaker; starts and `used` of both against the designed
    outcome and draw_reference on the exact tables."""
    render, R = _R()
    rng = np.random.default_rng(3601)
    k, designs, tail = residue_signal()
    N = len(k)
    loud = quantise(so.synth_dry(rng, N) * np.float32(6.0))
    src = DevPool([traj_beacon(rng, N)], levels="mono")
    d16 = R.dry_pool([k], levels=True, dtype="int16")
    df = R.dry_pool([to(values(k))], levels=True)
    dl = R.dry_pool([to(values(loud))], levels=True)
    check_tables(d16, 0, k, "residues")
    Tk, Tl = exact_table(k), exact_table(loud)
    U, M = len(designs), N - RW + 1
    zero = torch.zeros(1, dtype=torch.int32, device="cuda")
    u = to(np.array([[(s + 0.5) / M, (tail + 0.5) / M] for s, _, _, _ in designs]))
    got, plans = {}, []
    try:
        for arm, dres in (("i16", d16), ("float", df)):
            starts = torch.full((U,), -1, dtype=torch.int32, device="cuda")
            used = torch.full((U,), -7, dtype=torch.int32, device="cuda")
            outs = [torch.full((2, RW), NAN, device="cuda") for _ in range(2 * U)]
            srcs, draws = [], []
            for e in range(U):
                lanes = [dres, dl] if e % 2 == 0 else [dl, dres]
                srcs += [render.Pooled(src.pool, zero[0], (starts[e], RW), 0, render.DryPick(d, zero[0])) for d in lanes]
                draws.append(render.CropDraw(starts[e], [2 * e, 2 * e + 1], u[e], used[e]))
            plan = R.plan_device(srcs, outs, draws=draws)
            plans.append(plan)
            plan.run()
            assert _device_errors(R) == 0, arm
            got[arm] = (starts.cpu().numpy(), used.cpu().numpy(), torch.stack(outs).cpu().numpy())
        assert np.array_equal(got["i16"][0], got["float"][0]) and np.array_equal(got["i16"][1], got["float"][1])
        assert np.array_equal(got["i16"][2], got["float"][2])
        uh = u.cpu().numpy()
        counts = {kind: [0, 0] for kind in RES_KINDS}
        for e, (s, r, kind, is_loud) in enumerate(designs):
            want = (s, 1) if is_loud else (tail, 2)
            tabs = [Tk, Tl] if e % 2 == 0 else [Tl, Tk]
            assert dr.draw(tabs, [RW, RW], [N, N], RW, uh[e]) == want, (e, r, kind)
            assert dr.margins(tabs, [RW, RW], [N, N], RW, uh[e]) > 9.0, (e, r, kind)
            for arm in got:
                assert (int(got[arm][0][e]), int(got[arm][1][e])) == want, (arm, e, r, kind)
            counts[kind][int(is_loud)] += 1
        print("\nresidue draws: %d designed crops, every residue 0..63 at both crop ends; %s" % (U, counts))
    finally:
        for p in plans:
            p.close()
        for p in (d16, df, dl, src):
            p.close()


# ----------------------------------------------------------------------------------------- D. corpus size
D_SHORT = 3000                   # the first signal's shortfall from 2^23 samples
D_SHIFT = 997                    # signal i (i >= 1) is base[D_SHIFT * i:][:2^23]: every signal different
D_CONST = 200                    # the all -32768 signal


def corpus(n, gen):
    """n CUDA int16 signals: the first 2^23 - D_SHORT samples long, the others 2^23, views of one random full-range base
    tensor at different shifts, and signal D_CONST (when n > D_CONST) all -32768.  Returns (signals, base, offsets):
    signal i's byte offset in the pool's arena (each signal at a 64-byte boundary)."""
    M = 1 << 23
    base = torch.randint(-32768, 32768, (M + D_SHIFT * n,), dtype=torch.int16, device="cuda", generator=gen)
    sig = [base[:M - D_SHORT]] + [base[D_SHIFT * i:D_SHIFT * i + M] for i in range(1, n)]
    if n > D_CONST:
        sig[D_CONST] = torch.full((M,), -32768, dtype=torch.int16, device="cuda")
    off = np.concatenate([[0], np.cumsum([align_up(2 * x.numel(), 64) for x in sig])]).astype(np.int64)
    return sig, base, off


def straddling(off, at):
    """The signal whose bytes straddle byte offset `at`, and the sample of it at that offset."""
    i = int(np.searchsorted(off, at, side="right")) - 1
    assert off[i] < at < off[i + 1], (i, off[i], at)
    return i, (at - int(off[i])) // 2


@pytest.mark.parametrize("resident", ["device", "host"])
def test_corpus_size_pool(resident):
    render, R = _R()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3401)
    n = 257 if resident == "device" else 100
    sig, base, off = corpus(n, gen)
    torch.cuda.synchronize()
    R.reset_stats()
    ip = R.dry_pool(sig, levels=True, host=resident == "host", dtype="int16")
    launches = R.launch_count()
    rng = np.random.default_rng(3402)
    cands = [Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, B), np.round(np.linspace(0, N, P)).astype(np.int32))
             for N, P in ((40001, 3), (52002, 4))]
    pool = R.source_pool([c.src for c in cands])
    try:
        arena, tables = int(off[-1]), 8 * sum(-(-x.numel() // STRIDE) + 1 for x in sig)
        if resident == "device":
            assert arena > 1 << 32 and ip.nbytes == 8 * n + arena + 8 * n + tables and ip.host_nbytes == 0
            marks = [1 << 31, 1 << 32]
        else:
            assert ip.nbytes == 16 * n and ip.host_nbytes == arena + tables <= PINNED_MAX
            marks = [1 << 30, 3 << 29]
        # the signals that straddle each mark, their neighbours, the last signal and the all -32768 one
        # the layout from the pool's own signal addresses: each signal at a 64-byte boundary behind the last
        at = [R.lib.ss_dry_pool_signal_i16(ip._h, i) for i in range(n)]
        assert [a - at[0] for a in at] == [int(v) for v in off[:-1]], resident
        # the table build: per signal an expansion and a sparse sampling, and one k_levels per batch of expansions
        # (dry_copied_levels: batches of at most max(256 MiB, one signal) of float32 copies)
        cap, used, batches = max(STEM_BYTES, max(align_up(4 * x.numel(), 256) for x in sig)), 0, 1
        for x in sig:
            b = align_up(4 * x.numel(), 256)
            if used > 0 and used + b > cap:
                batches, used = batches + 1, 0
            used += b
        assert batches > 1 and launches == 2 * n + batches, (launches, n, batches)
        hold(ip)
        hit = [straddling(off, m) for m in marks]
        pick = sorted({j for i, _ in hit for j in (i - 1, i, i + 1) if j < n} | {0, n - 1} |
                      ({D_CONST} if n > D_CONST else set()))
        host = {i: sig[i].cpu().numpy() for i in pick}
        for i in pick:
            check_tables(ip, i, host[i], (resident, "corpus"))
        if n > D_CONST:
            t = ip.level_table(D_CONST).cpu().numpy()
            assert np.array_equal(t, np.arange(len(t), dtype=np.float64)), "all -32768: Q[s] = s"
        # stems and draws of slots that pick them, around the mark's sample
        wl = 6000
        slots = [(i, c, max(0, min(cands[c].N - wl, s - 1000 + 37 * c))) for i, s in hit for c in (0, 1)]
        slots += [(i, j % 2, 0) for j, i in enumerate(pick)]
        k = len(slots)
        vals = torch.tensor([[c for _, c, _ in slots], [i for i, _, _ in slots], [s for _, _, s in slots]],
                            dtype=torch.int32, device="cuda")
        outs = [Out(2, wl) for _ in range(k)]
        srcs = [render.Pooled(pool, vals[0, j], (vals[2, j], wl), 0, render.DryPick(ip, vals[1, j])) for j in range(k)]
        plan = R.plan_device(srcs, [o.view() for o in outs])
        du = torch.full((2, 5), 0.5, dtype=torch.float64, device="cuda")
        dst = torch.zeros(2, dtype=torch.int32, device="cuda")
        dused = torch.zeros(2, dtype=torch.int32, device="cuda")
        dv = torch.tensor([[0, 1], [hit[0][0], hit[-1][0]]], dtype=torch.int32, device="cuda")
        dsrc = [render.Pooled(pool, dv[0, j], (dst[j], wl), 0, render.DryPick(ip, dv[1, j])) for j in range(2)]
        douts = [Out(2, wl) for _ in range(2)]
        dplan = R.plan_device(dsrc, [o.view() for o in douts],
                              draws=[render.CropDraw(dst[j], [j], du[j], dused[j]) for j in range(2)])
        try:
            plan.run()
            dplan.run()
            torch.cuda.synchronize()
            R.check_device_errors()
            jobs = []
            for j, (i, c, s) in enumerate(slots):
                y = outs[j].get()
                xf = to(values(host[i]))
                ref = torch.empty((2, wl), device="cuda")
                R.render_device([cands[c].src._replace(dry=xf[:cands[c].N].contiguous(), window=(s, wl))], [ref])
                assert np.array_equal(y, ref.cpu().numpy()), (resident, j, i, s)
                jobs.append((ScaleCand(values(host[i])[:cands[c].N], cands[c].h, cands[c].b), y, s, wl, False,
                             "D corpus %s" % resident, "signal %d cand %d start %d" % (i, c, s)))
            ds, dus = dst.cpu().numpy(), dused.cpu().numpy()
            for j in range(2):
                i, c = int(dv[1, j]), j
                ref_t = exact_table(host[i])
                Nr = [cands[c].N]
                want = dr.draw([ref_t], [wl], Nr, wl, du[j].cpu().numpy())
                assert (int(ds[j]), int(dus[j])) == want, (resident, j, want)
                jobs.append((ScaleCand(values(host[i])[:cands[c].N], cands[c].h, cands[c].b), douts[j].get(),
                             int(ds[j]), wl, False, "D corpus %s" % resident, "drawn signal %d" % i))
            f64(jobs)
        finally:
            plan.close()
            dplan.close()
        print("\n%s corpus: %d signals, arena %d bytes (%.2f GiB), %d expansion batches, straddling signals %s, "
              "%d slots checked" % (resident, n, arena, arena / 2 ** 30, batches, hit, k))
        report("D corpus %s" % resident)
    finally:
        pool.close()
        ip.close()
        del sig, base
