"""Device plans at training scale against float64 (tests/render_reference.py, tests/mix_reference.py): moving crops,
direct stems and mixtures in chunks of many sources whose block tables k_blocks builds on the device.

- Source count per device-table chunk: one plan of 1 to 100 sources (whole stems, fixed and moving windows; bounds on
  the host, bounds on the device only, per-sample idx / w) in one chunk, so that k_blocks' loop past 8 sources and its
  work-item prefix past 32 run.  The plan runs 8 times with the starts rewritten on the stream in between; every stem
  of every run is checked sample by sample against float64 at its start.
- The training step at full scale: bench.py's 16 utterances, 2 banked speakers and 1 banked noise each, cropped to 4 s
  with one start per utterance, with a plain and a mono mixture per utterance, under the default chunk budget and in
  one chunk.
- Every kernel variant and every RIR flag set regrouped by arrange_chunks in one plan, reverberant and direct crops
  against float64, with mixtures whose stems cross the kinds.
- Out-of-range starts at scale: clamped, reported once as bit 2 of ss_device_errors, the other stems unchanged.

Every output lies inside a NaN-filled buffer with sentinels on both sides."""
import ctypes
import math

import numpy as np
import pytest
import torch

from chunk_budget import DEFAULT_CHUNK_BYTES, chunk_budget  # noqa: F401  (fixture)
from direct_path import direct_path_rirs, normalized
from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs, trajectory
from window_cases import full_blocks
from gpu_plumbing import _error_bits, _lib
from mix_reference import Out, PAD, check_mixture, fold

pytestmark = pytest.mark.gpu

B = 4096
ONE_CHUNK = 1 << 30             # a chunk budget that holds every batch of this file in one chunk per kernel variant
INT32_MIN, INT32_MAX = -2 ** 31, 2 ** 31 - 1
STATS = {}                      # label -> [worst local ratio, worst global relative RMS]


def _report(title):
    print("\n%s:" % title)
    for k in sorted(STATS):
        print("  %-22s worst per-sample ratio %.3g, worst global relative RMS %.3g" % (k, STATS[k][0], STATS[k][1]))


class Src:
    """One source: NumPy inputs for the float64 reference, device copies, an optional RIR bank, its outputs and its
    window ("whole", "fixed" or "moving").  kind: "fast" (aligned bounds on the host), "grid" (grid-blocked bounds,
    on the host or, with device_bounds, on the device only), "indexed" (per-sample idx / w), "long" (L > 4096, bounds
    on the host) or "static"."""

    def __init__(self, rng, kind, P, C, L, N, win="whole", n=0, fixed=0, banked=False, normalize=False, taps=0,
                 device_bounds=False, bounds=None, h=None):
        L_, R = _lib()
        self.kind, self.P, self.C, self.L, self.N = kind, P, C, L, N
        self.win, self.n, self.fixed = win, (n if win != "whole" else N), fixed
        self.banked, self.normalize, self.taps = banked, normalize, taps
        self.mode = {"static": 0, "indexed": 2}.get(kind, 1)
        self.x = so.synth_dry(rng, N)
        self.h = so.synth_rirs(rng, P, C, L) if h is None else h
        self.bounds = self.idx = self.w = None
        if self.mode == 1:
            self.bounds = np.ascontiguousarray(bounds, np.int32)
        elif self.mode == 2:
            idx, w = trajectory(bounds)
            self.idx, self.w, self.seg = idx.astype(np.int32), w, np.asarray(bounds, np.int64)
        self.h_ref = normalized(self.h) if normalize else self.h
        self.h_dir = direct_path_rirs(self.h_ref, taps) if taps else None
        to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()             # noqa: E731
        self.dx, self.dh = to(self.x), to(self.h)
        self.bank = R.rir_bank(self.dh, normalize=normalize, direct_taps=taps) if banked else None
        self.db = to(self.bounds) if self.mode == 1 else None
        self.bh = self.bounds if self.mode == 1 and not device_bounds else None
        self.di, self.dw = (to(self.idx), to(self.w)) if self.mode == 2 else (None, None)
        self.aligned = self._aligned()
        self.variant = "k_render<1,0>" if L > B else ("k_render_fast" if self.aligned or self.mode == 0
                                                      else "k_render<0,0>")
        self.out = Out(C, self.n)
        self.dout = Out(C, self.n) if taps else None

    def _aligned(self):
        """The blocking the library picks: the host's cost rule with bounds on the host, else aligned when the average
        segment is at least one block long."""
        if self.mode != 1 or self.L > B:
            return 0
        if self.bh is None:
            return int((self.P - 1) * B <= self.N)
        return host_aligned(self.bh, self.L, self.N)

    def item(self, start_ptr=None):
        L_, _ = _lib()
        flags = (L_.SS_RIR_NORMALIZE if self.normalize and not self.banked else 0) | \
            (L_.SS_DIRECT_TARGET if self.taps else 0)
        it = L_.SsSource(x=self.dx.data_ptr(), N=self.N, P=self.P, C=self.C, L=self.L, mode=self.mode, flags=flags,
                         out=self.out.ptr())
        if self.bank is not None:
            it.rir_bank = self.bank._h.value
        else:
            it.rir = self.dh.data_ptr()
        if self.taps:
            it.out_direct, it.direct_taps = self.dout.ptr(), self.taps
        if self.mode == 1:
            it.bounds = self.db.data_ptr()
            if self.bh is not None:
                it.bounds_host = self.bh.ctypes.data
        elif self.mode == 2:
            it.idx, it.w = self.di.data_ptr(), self.dw.data_ptr()
        if self.win == "fixed":
            it.win_len, it.win_start = self.n, self.fixed
        elif self.win == "moving":
            it.win_len, it.win_start_dev = self.n, start_ptr
        return it

    def outs(self):
        return [self.out] + ([self.dout] if self.dout is not None else [])

    def edges(self):
        """Block starts of the full plan and the waypoints, inside (0, N)."""
        blocks = full_blocks(self.N, self.bounds if self.mode == 1 else None, self.aligned)
        way = self.bounds if self.mode == 1 else (self.seg if self.mode == 2 else [])
        return sorted({int(b[0]) for b in blocks[1:]} | {int(v) for v in way if 0 < v < self.N})

    def start_classes(self, j, rng):
        """8 starts of the window: 0, N - n, an edge -1 / 0 / +1 for the first sample, another edge -1 / +1 for the last
        sample, and a random one; each kept inside [0, N - n]."""
        N, n = self.N, self.n
        e = self.edges() or [N // 2]
        e1, e2 = e[j % len(e)], e[(j * 5 + 3) % len(e)]
        v = [0, N - n, e1 - 1, e1, e1 + 1, e2 - n - 1, e2 - n + 1, int(rng.integers(0, N - n + 1))]
        return [min(max(s, 0), N - n) for s in v]

    def check(self, y, a, direct=False, label=""):
        """Sample by sample against float64 at window start a (a 0, n = N for a whole stem).  The relative RMS bound
        holds for crops of at least one block: the relative RMS of a few samples is their relative error, which is
        unbounded next to a zero crossing however small the error is against the sample's rounding scale."""
        h = self.h_dir if direct else self.h_ref
        y64, scale = render_check_inputs(self.x, h, self.mode, bounds=self.bounds, idx=self.idx, w=self.w,
                                         window=(a, self.n))
        long_crop = self.n >= B
        worst, g = check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL if long_crop else math.inf, n0=a, label=label)
        key = self.variant + (" direct" if direct else "")
        s = STATS.setdefault(key, [0.0, 0.0])
        s[0], s[1] = max(s[0], worst), max(s[1], g if long_crop else 0.0)

    def close(self):
        if self.bank is not None:
            self.bank.close()
            self.bank = None


def host_aligned(bounds, L, N):
    """The blocking the library picks for bounds on the host (ss_debug_plan, a host-only hook)."""
    L_, R = _lib()
    b = np.ascontiguousarray(bounds, np.int32)
    P = b.size
    it = L_.SsSource(x=1, rir=1, out=1, bounds=b.ctypes.data, N=N, P=P, C=1, L=L, mode=1, bounds_host=b.ctypes.data)
    cap = (N + B - 1) // B + P
    tab = np.zeros((cap, 4), np.int32)
    al = ctypes.c_int32()
    assert R.lib.ss_debug_plan(ctypes.byref(it), tab.ctypes.data, cap, ctypes.byref(al)) > 0
    return al.value


def _grid_bounds_host(rng, P, N):
    """Bounds whose short segments make the host's cost rule choose grid blocking (k_render<0,0>)."""
    s = int(rng.integers(1, N - 60 * (P - 2)))
    return np.array([0] + [s + 60 * k for k in range(P - 2)] + [N], np.int32)


def _random_bounds(rng, P, N):
    inner = np.sort(rng.choice(np.arange(1, N), P - 2, replace=False)) if P > 2 else []
    return np.array([0] + list(inner) + [N], np.int32)


def scale_sources(n, seed):
    """n small sources that all run k_render<0,0>, so that one budget puts them in one chunk: per-sample idx / w,
    grid-blocked bounds on the host and grid-blocked bounds on the device only, cycling against whole stems, fixed
    and moving windows; 3 of 4 banked, none normalised (3 launches per chunk)."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        kind = ("indexed", "host", "device")[i % 3]
        win = ("moving", "whole", "moving", "fixed", "moving")[i % 5]
        N = int(rng.integers(12000, 20001))
        C = int(rng.integers(1, 4))
        L = 1 if i % 7 == 0 else int(rng.integers(50, 601))
        if kind == "device":
            P = int(rng.integers(5, 7)) if N < 4 * B else 6           # (P - 1) * 4096 > N: grid blocking
            bounds = _random_bounds(rng, P, N)
        elif kind == "host":
            P = 6                          # four short segments: fewer or as few blocks make the aligned plan win
            for _ in range(100):
                bounds = _grid_bounds_host(rng, P, N)
                if not host_aligned(bounds, 600, N):
                    break
            assert not host_aligned(bounds, 600, N)
        else:
            P = int(rng.integers(2, 7))
            bounds = _random_bounds(rng, P, N)
        nwin = (1, B + 7, N // 3, int(rng.integers(2, N)))[i % 4]
        fixed = int(rng.integers(0, N - nwin + 1))
        out.append(Src(rng, "indexed" if kind == "indexed" else "grid", P, C, L, N, win, nwin, fixed,
                       banked=i % 4 != 3, device_bounds=kind == "device", bounds=bounds))
        assert out[-1].variant == "k_render<0,0>", (i, kind)
    return out


def _plan(items):
    L_, R = _lib()
    arr = (L_.SsSource * len(items))(*items)
    plan = ctypes.c_void_p()
    L_.check(R.lib.ss_plan_create(R.ctx, arr, len(items), ctypes.byref(plan)))
    return arr, plan


class Scale:
    """The plan of scale_sources(n): one int32 start per moving source."""

    def __init__(self, n, seed):
        self.srcs = scale_sources(n, seed)
        self.moving = [i for i, s in enumerate(self.srcs) if s.win == "moving"]
        self.starts = torch.zeros(max(len(self.moving), 1), dtype=torch.int32, device="cuda")
        slot = {i: k for k, i in enumerate(self.moving)}
        self.items = [s.item(self.starts[slot[i]].data_ptr() if i in slot else None) for i, s in enumerate(self.srcs)]
        self.arr, self.plan = _plan(self.items)

    def outs(self):
        return [o for s in self.srcs for o in s.outs()]

    def close(self):
        _lib()[1].lib.ss_plan_destroy(self.plan)
        for s in self.srcs:
            s.close()


N_SOURCES = [1, 8, 9, 24, 25, 32, 33, 64, 65, 100]


@pytest.mark.parametrize("n", N_SOURCES)
def test_device_table_chunk_of_n_sources(n, chunk_budget):
    L_, R = _lib()
    chunk_budget(ONE_CHUNK)
    _error_bits()
    sc = Scale(n, 100 + n)
    try:
        rng = np.random.default_rng(n)
        runs = 8
        table = np.zeros((runs, sc.starts.numel()), np.int32)
        for k, i in enumerate(sc.moving):
            table[:, k] = sc.srcs[i].start_classes(i, rng)
        d_table = torch.from_numpy(table).cuda()
        outs = sc.outs()
        c0 = R.launch_count()
        snaps = []
        for k in range(runs):                      # no host synchronise inside the loop
            sc.starts.copy_(d_table[k])
            for o in outs:
                o.reset()
            L_.check(R.lib.ss_plan_run(sc.plan, None))
            snaps.append([o.buf.clone() for o in outs])
        # one chunk: k_blocks, k_prepare, k_render<0,0> per run
        assert R.launch_count() - c0 == 3 * runs
        torch.cuda.synchronize()
        assert R.lib.ss_plan_is_graph(sc.plan) == 1
        for k in range(runs):
            for j, (s, o) in enumerate(zip(sc.srcs, outs)):
                y = o.get(snaps[k][j])
                if s.win == "moving":
                    a = int(table[k, sc.moving.index(j)])
                    s.check(y, a, label="n=%d source %d run %d start %d" % (n, j, k, a))
                elif k == 0:
                    s.check(y, s.fixed if s.win == "fixed" else 0, label="n=%d source %d (%s)" % (n, j, s.win))
                else:
                    assert torch.equal(snaps[k][j], snaps[0][j]), (n, j, k)
        # ss_render_dev on the same items writes the plan's bits
        for k in (0, runs - 1):
            sc.starts.copy_(d_table[k])
            for o in outs:
                o.reset()
            L_.check(R.lib.ss_render_dev(R.ctx, sc.arr, n, None))
            torch.cuda.synchronize()
            for j, o in enumerate(outs):
                assert torch.equal(o.buf, snaps[k][j]), ("ss_render_dev", n, j, k)
        assert _error_bits() == 0
        _report("%d sources in one device-table chunk" % n)
    finally:
        sc.close()


def test_clamped_starts_at_scale(chunk_budget):
    """The 65-source plan: starts -1, N - len + 1, INT32_MIN and INT32_MAX are clamped to 0 / N - len, reported once as
    bit 2 of ss_device_errors, and every other stem keeps its bits."""
    L_, R = _lib()
    chunk_budget(ONE_CHUNK)
    _error_bits()
    n = 65
    sc = Scale(n, 100 + n)
    try:
        rng = np.random.default_rng(7)
        valid = np.array([int(rng.integers(0, sc.srcs[i].N - sc.srcs[i].n + 1)) for i in sc.moving], np.int32)
        outs = sc.outs()
        sc.starts.copy_(torch.from_numpy(valid))
        L_.check(R.lib.ss_plan_run(sc.plan, None))
        before = [o.buf.clone() for o in outs]
        assert _error_bits() == 0
        bad = valid.copy()
        clamped = {}
        for q, k in enumerate(range(1, len(sc.moving), 3)):
            s = sc.srcs[sc.moving[k]]
            v = (-1, s.N - s.n + 1, INT32_MIN, INT32_MAX)[q % 4]
            bad[k] = v
            clamped[sc.moving[k]] = 0 if v < 0 else s.N - s.n
        assert len(clamped) >= 8 and max(clamped) >= 32
        sc.starts.copy_(torch.from_numpy(bad))
        for o in outs:
            o.reset()
        L_.check(R.lib.ss_plan_run(sc.plan, None))
        assert _error_bits() == 4                               # reported once ...
        assert _error_bits() == 0                               # ... and cleared by the read
        for j, (s, o) in enumerate(zip(sc.srcs, outs)):
            if j in clamped:
                s.check(o.get(), clamped[j], label="clamped source %d" % j)
            else:
                o.get()
                assert torch.equal(o.buf, before[j]), j
        _report("clamped starts, 65 sources")
    finally:
        sc.close()


# ------------------------------------------------------------------------------------------------ mixtures


class PlanMix:
    """One ss_plan_mix over guarded outputs: mix (T,) or (C, T), speakers_out (S, ...), rms_db (S,)."""

    def __init__(self, speakers, noises, C, T, mono, sirs, snr):
        L_, _ = _lib()
        self.speakers, self.noises, self.mono = list(speakers), list(noises), mono
        S, rows = len(speakers), 1 if mono else C
        self.mix, self.out, self.rms = Out(rows, T), Out(S * rows, T), Out(1, S)
        self.sirs, self.snr = sirs, snr
        e = L_.SsPlanMix(S=S, M=len(noises), sirs=sirs.data_ptr() if S > 1 else None, snr=snr.data_ptr(),
                         mix=self.mix.ptr(), speakers_out=self.out.ptr(), rms_db=self.rms.ptr(),
                         flags=L_.SS_MIX_MONO if mono else 0)
        for i, v in enumerate(speakers):
            e.speakers[i] = v
        for i, v in enumerate(noises):
            e.noises[i] = v
        self.entry = e

    def bufs(self):
        return [self.mix, self.out, self.rms]

    def check(self, stems, snap, sirs, snr, label):
        """stems: every source's (C, T) output of this run; snap: snapshots of bufs()."""
        f = (lambda a: fold(a)) if self.mono else (lambda a: a.reshape(-1))             # noqa: E731
        spk = np.stack([f(stems[i]) for i in self.speakers])
        noi = np.stack([f(stems[i]) for i in self.noises])
        mix, out, rms = (b.get(s) for b, s in zip(self.bufs(), snap))
        check_mixture(spk, noi, sirs, snr, mix.reshape(-1), out.reshape(len(self.speakers), -1), rms.reshape(-1),
                      label)


# ------------------------------------------------------------------------------------------------ kinds and flags
def _kind_source(rng, kind, flagset, C, N, T):
    normalize, taps, banked = {"norm": (True, 0, False), "direct": (False, 40, False), "bank": (True, 40, True)}[flagset]
    if kind == "fast":
        P, L, bounds = 4, 600, np.array([0, 6000, 12500, N], np.int32)
    elif kind == "grid":
        P, L, bounds = 6, 600, _random_bounds(rng, 6, N)
    elif kind == "indexed":
        P, L, bounds = 5, 600, _random_bounds(rng, 5, N)
    elif kind == "long":
        P, L, bounds = 4, 5000, np.array([0, 4000, 11000, N], np.int32)
    else:
        P, L, bounds = 1, 900, None
    h = so.synth_rirs(rng, P, C, L)
    if kind == "long":                                   # a peak in the second partition
        h[-1, -1, 4500] = np.float32(3.0) * np.abs(h).max()
    return Src(rng, kind, P, C, L, N, "moving", T, banked=banked, normalize=normalize, taps=taps,
               device_bounds=kind == "grid", bounds=bounds, h=h)


KIND_VARIANT = {"fast": "k_render_fast", "static": "k_render_fast", "grid": "k_render<0,0>",
                "indexed": "k_render<0,0>", "long": "k_render<1,0>"}


def test_kinds_and_flags_regrouped_in_one_plan(chunk_budget):
    """fast, grid, indexed and long moving sources and static ones, each raw with SS_RIR_NORMALIZE, raw with
    SS_DIRECT_TARGET and banked with both, listed kind by kind inside each flag set (so arrange_chunks regroups them),
    each with its own moving start; mixtures whose stems cross the kinds.  Three runs with new starts, SIRs and SNRs:
    every reverberant and direct crop against float64 of the (normalised, cut) RIRs, every mixture against
    mix_reference."""
    L_, R = _lib()
    chunk_budget(ONE_CHUNK)
    _error_bits()
    rng = np.random.default_rng(31)
    C, N, T = 2, 20000, 5000
    order = [(k, f) for f in ("norm", "direct", "bank") for k in ("grid", "fast", "long", "static", "indexed")]
    srcs = [_kind_source(rng, k, f, C, N, T) for k, f in order]
    for s, (k, _) in zip(srcs, order):
        assert s.variant == KIND_VARIANT[k], (k, s.variant)
    ix = {kf: i for i, kf in enumerate(order)}
    starts = torch.zeros(len(srcs), dtype=torch.int32, device="cuda")
    sirs = torch.zeros((4, 2), device="cuda")
    snr = torch.zeros(4, device="cuda")
    mixes = [PlanMix([ix["fast", "norm"], ix["grid", "direct"], ix["long", "bank"]], [ix["static", "direct"]], C, T,
                     False, sirs[0], snr[0:1]),
             PlanMix([ix["indexed", "bank"], ix["long", "norm"]], [ix["static", "bank"], ix["fast", "direct"]], C, T,
                     True, sirs[1], snr[1:2]),
             PlanMix([ix["long", "direct"]], [ix["indexed", "norm"]], C, T, False, sirs[2], snr[2:3]),
             PlanMix([ix["static", "norm"], ix["grid", "bank"], ix["indexed", "direct"]],
                     [ix["grid", "norm"], ix["fast", "bank"]], C, T, True, sirs[3], snr[3:4])]
    items = [s.item(starts[i].data_ptr()) for i, s in enumerate(srcs)]
    arr = (L_.SsSource * len(items))(*items)
    marr = (L_.SsPlanMix * len(mixes))(*[m.entry for m in mixes])
    plan = ctypes.c_void_p()
    L_.check(R.lib.ss_plan_create_mix(R.ctx, arr, len(items), marr, len(mixes), ctypes.byref(plan)))
    try:
        g = torch.Generator(device="cuda")
        g.manual_seed(31)
        outs = [o for s in srcs for o in s.outs()]
        mbufs = [b for m in mixes for b in m.bufs()]
        hi = torch.tensor([N - T], dtype=torch.int32, device="cuda")
        runs, snaps = 3, []
        c0 = R.launch_count()
        for k in range(runs):
            starts.copy_(torch.randint(0, N - T + 1, (len(srcs),), dtype=torch.int32, device="cuda", generator=g))
            if k == 0:
                starts[:5].zero_()
                starts[5:10].copy_(hi.expand(5))
            sirs.uniform_(-6, 6, generator=g)
            snr.uniform_(10, 20, generator=g)
            for o in outs + mbufs:
                o.reset()
            L_.check(R.lib.ss_plan_run(plan, None))
            snaps.append([x.clone() for x in (starts, sirs, snr)] + [o.buf.clone() for o in outs + mbufs])
        # three chunks (one per kernel variant), each k_blocks, k_rir_absmax, k_rir_direct, k_prepare and the render;
        # then the four mixture kernels
        assert R.launch_count() - c0 == runs * (3 * 5 + 4)
        torch.cuda.synchronize()
        assert R.lib.ss_plan_is_graph(plan) == 1
        for k, sn in enumerate(snaps):
            st, sr_, sn_ = (t.cpu().numpy() for t in sn[:3])
            bufs = sn[3:]
            stems, j = [], 0
            for i, s in enumerate(srcs):
                a = int(st[i])
                y = s.out.get(bufs[j])
                s.check(y, a, label="%s/%s run %d start %d" % (order[i] + (k, a)))
                stems.append(y)
                j += 1
                if s.dout is not None:
                    s.check(s.dout.get(bufs[j]), a, direct=True, label="%s/%s direct run %d start %d" % (order[i] + (k, a)))
                    j += 1
            for q, m in enumerate(mixes):
                m.check(stems, bufs[j:j + 3], sr_[q], sn_[q], "mixture %d run %d" % (q, k))
                j += 3
        assert _error_bits() == 0
        _report("kinds and flags regrouped in one plan")
    finally:
        R.lib.ss_plan_destroy(plan)
        for s in srcs:
            s.close()


# ------------------------------------------------------------------------------------------------ training step
@pytest.mark.parametrize("budget", ["default", "one-chunk"])
def test_training_step_at_full_scale(budget, chunk_budget):
    """bench.py's 16 utterances (2 banked configs[1] speakers each) plus one banked static noise each, cropped to 4 s with
    one start per utterance, one plain and one mono Mixture per utterance: 48 sources, 32 mixtures.  Three steps with
    new starts (the first includes 0 and N - T), SIRs and SNRs: every crop against float64 and bit-equal to the same
    slice of its full stem from a separate whole-stem plan; every mixture against mix_reference.  The launch count
    gives the number of chunks; under the one-chunk budget all 48 sources share one k_blocks CTA."""
    import bench
    from sonicsim_b200 import render
    R = chunk_budget(DEFAULT_CHUNK_BYTES)
    _error_bits()
    U, T = 16, 4 * 16000
    C, N, S = bench.CFG["C"], bench.CFG["N"], bench.CFG["speakers"]
    items = bench.make_inputs(U, 0)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()                     # noqa: E731
    rng = np.random.default_rng(5)
    data, banks, srcs = [], [], []                                          # data: (x, h (P, C, L), bounds or None)
    for u in range(U):
        for k in range(S):
            x, h, b = items[S * u + k]
            data.append((x, h, b))
        x = (rng.standard_normal(N) * 0.05).astype(np.float32)
        h = (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32)
        data.append((x, h[None], None))
    starts = torch.zeros(U, dtype=torch.int32, device="cuda")
    sirs = torch.zeros((U, S - 1), device="cuda")
    snr = torch.zeros(U, device="cuda")
    for i, (x, h, b) in enumerate(data):
        u = i // (S + 1)
        if b is not None:
            bk = R.rir_bank(to(h))
            srcs.append(render.MovingSource(to(x), bk, to(b), b, window=(starts[u], T)))
        else:
            bk = R.rir_bank(to(h[0]))
            srcs.append(render.StaticSource(to(x), bk, window=(starts[u], T)))
        banks.append(bk)
    full = [torch.empty((C, N), device="cuda") for _ in srcs]
    p_full = R.plan_device([s._replace(window=None) for s in srcs], full)
    p_full.run()

    if budget == "one-chunk":
        R.set_chunk_bytes(ONE_CHUNK)
    stems = [Out(C, T) for _ in srcs]
    mixes = []
    for u in range(U):
        spk = [(S + 1) * u + k for k in range(S)]
        for mono in (False, True):
            rows = 1 if mono else C
            m = (Out(rows, T), Out(S * rows, T), Out(1, S))
            mixes.append((spk, [(S + 1) * u + S], mono, m,
                          render.Mixture(spk, [(S + 1) * u + S], sirs[u], snr[u], m[0].view(*((T,) if mono else (C, T))),
                                         m[1].view(*((S, T) if mono else (S, C, T))), m[2].view(S), mono)))
    plan = R.plan_device(srcs, [o.view() for o in stems], mixtures=[m[4] for m in mixes])
    try:
        g = torch.Generator(device="cuda")
        g.manual_seed(2024)
        edge = torch.tensor([0, N - T], dtype=torch.int32, device="cuda")
        bufs = stems + [b for m in mixes for b in m[3]]
        snaps = []
        c0 = R.launch_count()
        for k in range(3):                                                  # no host synchronise inside the loop
            starts.copy_(torch.randint(0, N - T + 1, (U,), dtype=torch.int32, device="cuda", generator=g))
            if k == 0:
                starts[:2].copy_(edge)
            sirs.uniform_(-6, 6, generator=g)
            snr.uniform_(10, 20, generator=g)
            for o in bufs:
                o.reset()
            plan.run()
            snaps.append([x.clone() for x in (starts, sirs, snr)] + [o.buf.clone() for o in bufs])
        launches = (R.launch_count() - c0) // 3
        chunks = (launches - 4) / 3
        print("\n%s budget: %d launches per step, %g chunks for 48 banked 4 s crops" % (budget, launches, chunks))
        assert chunks == int(chunks) and chunks >= 1
        if budget == "one-chunk":
            assert chunks == 1
        torch.cuda.synchronize()
        assert plan.is_graph()
        for k, sn in enumerate(snaps):
            st, sr_, sn_ = (t.cpu().numpy() for t in sn[:3])
            crops = []
            for i, ((x, h, b), o) in enumerate(zip(data, stems)):
                a = int(st[i // (S + 1)])
                assert torch.equal(sn[3 + i][PAD:-PAD].view(C, T), full[i][:, a:a + T]), (k, i, a)
                y = o.get(sn[3 + i])
                y64, scale = render_check_inputs(x, h, 1 if b is not None else 0, bounds=b, window=(a, T))
                worst, gl = check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=a,
                                         label="step %d source %d start %d" % (k, i, a))
                key = "train k_render_fast"
                s_ = STATS.setdefault(key, [0.0, 0.0])
                s_[0], s_[1] = max(s_[0], worst), max(s_[1], gl)
                crops.append(y)
            j = 3 + len(stems)
            for q, (spk, noi, mono, m, _) in enumerate(mixes):
                u = q // 2
                f = (lambda a: fold(a)) if mono else (lambda a: a.reshape(-1))           # noqa: E731
                mix, out, rms = (b_.get(s) for b_, s in zip(m, sn[j:j + 3]))
                check_mixture(np.stack([f(crops[i]) for i in spk]), np.stack([f(crops[i]) for i in noi]), sr_[u],
                              sn_[u], mix.reshape(-1), out.reshape(S, -1), rms.reshape(-1),
                              "utterance %d mono %s step %d" % (u, mono, k))
                j += 3
        R.check_device_errors()
        _report("training step, %s budget" % budget)
    finally:
        plan.close()
        p_full.close()
        for bk in banks:
            bk.close()
