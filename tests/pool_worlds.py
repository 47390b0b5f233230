"""Candidates, pools, slots and training plans that the GPU pool and dry-pool tests build their worlds from.  Test
infrastructure."""
import ctypes
import threading

import numpy as np
import pytest
import torch

import draw_reference as dr
from direct_path import direct_path_rirs, normalized
from draw_reference import LEN, NEAR_DB, RATE, gappy_dry
from gpu_plumbing import _R, _device_errors, _rms, pmap, to
from mix_reference import Out, check_mixture, fold
from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, delay_rirs, graded_dry, render_check_inputs
from window_cases import _choice, stage_set_np

B = 4096
NAN = float("nan")
TRIES = 101                    # tries of the training plans' CropDraws
PINNED_MAX = 2 << 30           # pinned host bytes a scale test may hold in banks and pools


def fold_dev(t):
    """SS_MIX_MONO's channel mean of a (C, T) tensor, in NumPy: float32 sum in channel order, then an IEEE division by C."""
    a = t.cpu().numpy()
    acc = a[0].copy()
    for c in range(1, a.shape[0]):
        acc = acc + a[c]
    return torch.from_numpy(acc / np.float32(a.shape[0])).cuda()

TAPS = 40


class Cand:
    """One candidate: host inputs, its banked source and its full stem(s) rendered by ss_render_dev."""

    def __init__(self, x, h, b, taps=0):
        render, R = _R()
        self.x, self.h, self.b, self.N = x, h, b, len(x)
        self.C, self.L = h.shape[-2], h.shape[-1]
        self.bank = R.rir_bank(to(h), direct_taps=taps)
        self.src = (render.MovingSource(to(x), self.bank, to(b), b) if b is not None
                    else render.StaticSource(to(x), self.bank))
        self.full = torch.empty((self.C, self.N), device="cuda")
        self.full_d = torch.empty((self.C, self.N), device="cuda") if taps else None
        R.render_device([self.src._replace(direct_taps=taps)], [self.full],
                        direct_outs=[self.full_d] if taps else None)


def speakers(seed, n=5, C=2, taps=TAPS):
    """Moving candidates with a few long segments (aligned blocking on their own), all different P and N."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        P, N = 3 + j % 3, 30000 + 4099 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        assert _choice(b, N, P, 4096) == 1
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, C, 4096), b, taps))
    return out


def noises(seed, n=4, C=2):
    rng = np.random.default_rng(seed)
    return [Cand(so.synth_dry(rng, 26000 + 3001 * j), so.synth_rirs(rng, 1, C, 4096)[0], None) for j in range(n)]


def longs(seed, n=3):
    """Moving candidates with L > 4096 (K = 3): grid blocking, k_render<LONG>."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        P, N = 3 + j % 2, 24000 + 5003 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 1, 9000), b))
    return out


class PooledSlots:
    """k pooled slots over one pool with device starts, plus one with a fixed start; NaN-filled outputs."""

    def __init__(self, pool, cands, wl, k=4, fixed=123, taps=0):
        render, _ = _R()
        self.pool, self.cands, self.wl, self.fixed, self.taps = pool, cands, wl, fixed, taps
        self.picks = torch.zeros(k + 1, dtype=torch.int32, device="cuda")
        self.starts = torch.zeros(k, dtype=torch.int32, device="cuda")
        self.srcs = [render.Pooled(pool, self.picks[j], (self.starts[j], wl), taps) for j in range(k)]
        self.srcs.append(render.Pooled(pool, self.picks[k], (fixed, wl), taps))
        C = cands[0].C
        self.outs = [torch.empty((C, wl), device="cuda") for _ in self.srcs]
        self.douts = [torch.empty((C, wl), device="cuda") for _ in self.srcs] if taps else None

    def draw(self, rng, pk=None, st=None):
        n = len(self.cands)
        pk = rng.integers(0, n, len(self.srcs)) if pk is None else np.asarray(pk)
        if st is None:
            st = [int(rng.integers(0, self.cands[p].N - self.wl + 1)) for p in pk[:-1]]
        self.pk, self.st = [int(v) for v in pk], [int(v) for v in st] + [self.fixed]
        self.picks.copy_(torch.tensor(self.pk, dtype=torch.int32))
        self.starts.copy_(torch.tensor(self.st[:-1], dtype=torch.int32))
        for o in self.outs + (self.douts or []):
            o.fill_(NAN)

    def check(self, what):
        """Every output against ss_render_dev of the picked candidate with a fixed window, and the full stem's slice."""
        _, R = _R()
        refs = [torch.empty_like(o) for o in self.outs]
        drefs = [torch.empty_like(o) for o in self.outs] if self.taps else None
        R.render_device([self.cands[p].src._replace(window=(a, self.wl), direct_taps=self.taps)
                         for p, a in zip(self.pk, self.st)], refs, direct_outs=drefs)
        torch.cuda.synchronize()
        for j, (p, a) in enumerate(zip(self.pk, self.st)):
            c = self.cands[p]
            assert torch.equal(self.outs[j], refs[j]), (what, j, p, a)
            assert torch.equal(self.outs[j], c.full[:, a:a + self.wl]), (what, j, p, a)
            if self.taps:
                assert torch.equal(self.douts[j], drefs[j]), (what, "direct", j, p, a)
                assert torch.equal(self.douts[j], c.full_d[:, a:a + self.wl]), (what, "direct", j, p, a)


def _mix_dev(R, spk, noi, sirs, snr):
    """ss_mix_dev on stems already folded: spk (S, T), noi (M, T) -> mix (T,), speakers after their gains (S, T)."""
    from sonicsim_b200 import _lib
    S, M = spk.shape[0], noi.shape[0]
    spk, noi = spk.contiguous().clone(), noi.contiguous()
    mix = torch.empty(spk.shape[1], device="cuda")
    scr = torch.empty(int(R.lib.ss_mix_scratch_doubles()), dtype=torch.float64, device="cuda")
    it = _lib.SsMixItem(speakers=spk.data_ptr(), noises=noi.data_ptr(), sirs=sirs.data_ptr(), mix=mix.data_ptr(),
                        speakers_out=spk.data_ptr(), scratch=scr.data_ptr(), E=spk.shape[1], S=S, M=M,
                        snr=float(snr.item()))
    _lib.check(R.lib.ss_mix_dev(R.ctx, ctypes.byref(it), 1, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return mix, spk


def _training_plan(R, render, spk_pool, noi_pool, U, S, T):
    """U scenes: S pooled speakers and one pooled noise each, one device start per scene, one mono Mixture each."""
    picks = torch.zeros((U, S), dtype=torch.int32, device="cuda")
    scene = torch.zeros(U, dtype=torch.int32, device="cuda")
    starts = torch.zeros(U, dtype=torch.int32, device="cuda")
    sirs = torch.zeros((U, S - 1), device="cuda")
    snr = torch.zeros(U, device="cuda")
    srcs, outs = [], []
    C = spk_pool.C
    for u in range(U):
        srcs += [render.Pooled(spk_pool, picks[u, k], (starts[u], T)) for k in range(S)]
        srcs.append(render.Pooled(noi_pool, scene[u], (starts[u], T)))
        outs += [torch.empty((C, T), device="cuda") for _ in range(S + 1)]
    mix = torch.empty((U, T), device="cuda")
    spk_out = torch.empty((U, S, T), device="cuda")
    rms = torch.empty((U, S), device="cuda")
    mixtures = [render.Mixture(list(range((S + 1) * u, (S + 1) * u + S)), [(S + 1) * u + S], sirs[u], snr[u], mix[u],
                               spk_out[u], rms[u], mono=True) for u in range(U)]
    plan = R.plan_device(srcs, outs, mixtures=mixtures)
    return plan, dict(picks=picks, scene=scene, starts=starts, sirs=sirs, snr=snr, outs=outs, mix=mix,
                      spk_out=spk_out, rms=rms)


def _draw_training(st, n_scenes, S, n_min, T, g):
    U = st["scene"].numel()
    sc = torch.randint(0, n_scenes, (U,), device="cuda", dtype=torch.int32, generator=g)
    st["picks"].copy_(S * sc[:, None] + torch.rand(U, S, device="cuda", generator=g).argsort(1).int())
    st["scene"].copy_(sc)
    st["starts"].copy_(torch.randint(0, n_min - T + 1, (U,), device="cuda", dtype=torch.int32, generator=g))
    st["sirs"].uniform_(-6, 6, generator=g)
    st["snr"].uniform_(10, 20, generator=g)


def moving(seed, Ls, taps=0, aligned=None):
    rng = np.random.default_rng(seed)
    out = []
    for j, L in enumerate(Ls):
        P, N = 3 + j % 3, 30000 + 4099 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        if aligned is not None:
            assert _choice(b, N, P, L) == aligned, (L, P, N)
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, L), b, taps))
    return out


def dry_signals(seed, n, length, tail):
    """n dry signals of `length` finite samples followed by `tail` NaNs (never read by a slot)."""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        x = np.full(length + tail, np.nan, np.float32)
        x[:length] = so.synth_dry(rng, length)
        out.append(to(x))
    return out


@pytest.fixture(scope="module")
def world():
    spk = speakers(301, n=4, taps=TAPS)                       # aligned moving, direct sets
    lng = moving(302, [5000, 9000, 13000, 6000])              # K = 2, 3, 4, 2: grid, k_render<LONG>
    noi = noises(303, n=3)                                    # static
    return {"speakers": (spk, TAPS), "long": (lng, 0), "noise": (noi, 0)}


def reference(c, x, s, wl, taps):
    """render_device of candidate c with dry x[:N] (a contiguous copy) at the fixed window (s, wl)."""
    render, R = _R()
    out = torch.empty((c.C, wl), device="cuda")
    dout = torch.empty((c.C, wl), device="cuda") if taps else None
    R.render_device([c.src._replace(dry=x[:c.N].contiguous(), window=(s, wl), direct_taps=taps)], [out],
                    direct_outs=[dout] if taps else None)
    return out, dout


class DrySlots:
    """k dry-picked pooled slots over one pool, each with its own pick, dry pick and start tensor; NaN-filled outputs."""

    def __init__(self, pool, dpool, cands, wl, taps, k=4, dry=True):
        render, _ = _R()
        self.cands, self.wl, self.taps, self.k = cands, wl, taps, k
        self.picks = torch.zeros(k, dtype=torch.int32, device="cuda")
        self.dpicks = torch.zeros(k, dtype=torch.int32, device="cuda")
        self.starts = torch.zeros(k, dtype=torch.int32, device="cuda")
        C = cands[0].C
        self.outs = [torch.empty((C, wl), device="cuda") for _ in range(k)]
        self.douts = [torch.empty((C, wl), device="cuda") for _ in range(k)] if taps else None
        self.srcs = [render.Pooled(pool, self.picks[j], (self.starts[j], wl), taps,
                                   render.DryPick(dpool, self.dpicks[j]) if dry else None) for j in range(k)]

    def fill(self, gen, n, n_dry, n_min):
        self.picks.copy_(torch.randint(0, n, (self.k,), generator=gen, device="cuda", dtype=torch.int32))
        self.dpicks.copy_(torch.randint(0, n_dry, (self.k,), generator=gen, device="cuda", dtype=torch.int32))
        self.starts.copy_(torch.randint(0, n_min - self.wl + 1, (self.k,), generator=gen, device="cuda",
                                        dtype=torch.int32))
        for o in self.outs + (self.douts or []):
            o.fill_(NAN)

    def snap(self):
        return dict(picks=self.picks.clone(), dpicks=self.dpicks.clone(), starts=self.starts.clone(),
                    outs=[o.clone() for o in self.outs], douts=[o.clone() for o in self.douts or []])

    def check(self, snap, signals, what):
        for j in range(self.k):
            c = self.cands[int(snap["picks"][j])]
            x = signals[int(snap["dpicks"][j])]
            s = int(snap["starts"][j])
            ref, dref = reference(c, x, s, self.wl, self.taps)
            y = snap["outs"][j]
            assert torch.isfinite(y).all(), (what, j)
            assert torch.equal(y, ref), (what, j, int(snap["picks"][j]), int(snap["dpicks"][j]), s)
            if self.taps:
                assert torch.isfinite(snap["douts"][j]).all() and torch.equal(snap["douts"][j], dref), (what, j)


@pytest.fixture(scope="module")
def draw_world():
    """Moving speakers of 12.5 to 20 s (aligned, levels "mono" for the speaker without a dry pick), static noises, and
    gappy dry streams of 26 s."""
    rng = np.random.default_rng(321)
    spk = []
    for j in range(4):
        P, N = 3 + j % 3, 200000 + 37003 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        spk.append(Cand(gappy_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    noi = [Cand(so.synth_dry(rng, 180000 + 51001 * j), so.synth_rirs(rng, 1, 2, 4096)[0], None) for j in range(3)]
    dry = [gappy_dry(rng, 26 * RATE) for _ in range(6)]
    return spk, noi, dry


class DrawStep:
    """B examples: speaker 0 dry-picked, speaker 1 dry-picked or not (`mixed`), a pooled noise; one CropDraw each."""

    def __init__(self, R, render, sp, npool, dpool, B, mixed=True, thr=-40.0, tries=101, dry=True):
        d = "cuda"
        self.B, self.mixed, self.thr = B, mixed, thr
        self.picks = torch.zeros((B, 3), dtype=torch.int32, device=d)
        self.dpicks = torch.zeros((B, 2), dtype=torch.int32, device=d)
        self.starts = torch.zeros(B, dtype=torch.int32, device=d)
        self.u = torch.zeros((B, tries), dtype=torch.float64, device=d)
        self.used = torch.full((B,), -7, dtype=torch.int32, device=d)
        self.outs = [torch.empty((2, LEN), device=d) for _ in range(3 * B)]
        self.srcs, self.draws = [], []
        for b in range(B):
            dp0 = render.DryPick(dpool, self.dpicks[b, 0]) if dry else None
            dp1 = render.DryPick(dpool, self.dpicks[b, 1]) if dry and not mixed else None
            self.srcs += [render.Pooled(sp, self.picks[b, 0], (self.starts[b], LEN), 0, dp0),
                          render.Pooled(sp, self.picks[b, 1], (self.starts[b], LEN), 0, dp1),
                          render.Pooled(npool, self.picks[b, 2], (self.starts[b], LEN))]
            self.draws.append(render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], self.u[b], self.used[b], thr))
        self.plan = R.plan_device(self.srcs, self.outs, draws=self.draws)

    def fill(self, gen, ns, nn, nd):
        self.picks[:, :2].copy_(torch.randint(0, ns, (self.B, 2), generator=gen, device="cuda", dtype=torch.int32))
        self.picks[:, 2].copy_(torch.randint(0, nn, (self.B,), generator=gen, device="cuda", dtype=torch.int32))
        self.dpicks.copy_(torch.randint(0, nd, (self.B, 2), generator=gen, device="cuda", dtype=torch.int32))
        self.u.uniform_(generator=gen)
        for o in self.outs:
            o.fill_(NAN)

    def snap(self):
        return dict(picks=self.picks.clone(), dpicks=self.dpicks.clone(), starts=self.starts.clone(),
                    used=self.used.clone(), u=self.u.clone(), outs=[o.clone() for o in self.outs])

    def check(self, snap, spk, noi, dry_dev, Tp, Td, what, stems=True):
        """Every example against draw_reference on the device's tables; returns (checked, near)."""
        picks, dpicks = snap["picks"].cpu().numpy(), snap["dpicks"].cpu().numpy()
        starts, used, u = snap["starts"].cpu().numpy(), snap["used"].cpu().numpy(), snap["u"].cpu().numpy()
        checked = near = 0
        for b in range(self.B):
            p0, p1, pn = (int(v) for v in picks[b])
            d0, d1 = (int(v) for v in dpicks[b])
            Nr = [spk[p0].N, spk[p1].N, noi[pn].N]
            tabs = [Td[d0], Tp[p1] if self.mixed else Td[d1]]
            s, k = int(starts[b]), int(used[b])
            assert 0 <= s <= min(Nr) - LEN, (what, b, s, Nr)
            if stems:
                for j, (c, x) in enumerate(((spk[p0], dry_dev[d0]), (spk[p1], None if self.mixed else dry_dev[d1]),
                                            (noi[pn], None))):
                    want = reference(c, x, s, LEN, 0)[0] if x is not None else c.full[:, s:s + LEN]
                    assert torch.equal(snap["outs"][3 * b + j], want), (what, b, j)
            if dr.margins(tabs, [LEN, LEN], Nr, LEN, u[b], self.thr) < NEAR_DB:
                near += 1
                continue
            assert (s, k) == dr.draw(tabs, [LEN, LEN], Nr, LEN, u[b], self.thr), (what, b, Nr)
            checked += 1
        return checked, near


def _host_pool(R, render, cands, taps=0, levels=None, lufs=None):
    """The candidates over host banks, NumPy dry signals and bounds: the pool copies them."""
    out = []
    for c in cands:
        bank = R.rir_bank(c.h, direct_taps=taps, host=True)
        out.append(render.MovingSource(c.x, bank, c.b, c.b) if c.b is not None else render.StaticSource(c.x, bank))
    return R.source_pool(out, levels=levels, lufs_targets=lufs)


def host_src(render, c, taps=0):
    """The candidate as a host-path source over the same bank."""
    if c.b is None:
        return render.StaticSource(c.x, c.bank, direct_taps=taps)
    return render.MovingSource(c.x, c.bank, c.b, direct_taps=taps)


def gain_pool(R, render, cands, targets, taps=0, levels=None):
    pool = R.source_pool([c.src for c in cands], levels=levels, lufs_targets=targets, sr=RATE)
    norm = [NCand(c, *normalised(R, render, c, t, taps)) if t is not None else NCand(c, c.full, c.full_d, None)
            for c, t in zip(cands, targets)]
    return pool, norm

STEM_BYTES = 256 << 20         # the transient stem buffer of the pool builds (kLevelStemBytes)


def align_up(v, a):
    return (v + a - 1) // a * a


def stem_groups(C, Ns):
    """The grouping of the pool builds restated: candidate i takes align_up(4 C N_i, 256) bytes of a buffer of
    max(256 MiB, largest stem) bytes, and a candidate that does not fit behind the group's others starts a new group.
    Returns (first candidate of every group + [n], buffer bytes)."""
    b = [align_up(4 * C * N, 256) for N in Ns]
    cap = max(STEM_BYTES, max(b))
    first, used = [0], 0
    for i, v in enumerate(b):
        if used > 0 and used + v > cap:
            first.append(i)
            used = 0
        used += v
    return first + [len(Ns)], cap


def table_error(q, y, mono):
    """|Q - Q_ref| / Q_ref[N] of a device table against the long-double prefix of stem y (0 when both are 0)."""
    ref = dr.level_table(y, mono, np.longdouble)
    assert q.shape == ref.shape and q[0] == 0.0
    err = float(np.max(np.abs(q.astype(np.longdouble) - ref)))
    top = float(ref[-1])
    if top == 0.0:
        assert err == 0.0
        return 0.0
    return err / top


class ScaleCand:
    """One candidate: dry x (N,), RIRs h (P, C, L) (P = 1: static), bounds (P,) or None, K partitions."""

    def __init__(self, x, h, b):
        self.x, self.h, self.b = np.ascontiguousarray(x, np.float32), np.ascontiguousarray(h, np.float32), b
        self.N, (self.P, self.C, self.L) = len(x), h.shape
        self.K = (self.L + B - 1) // B
        self.mode = 0 if b is None else 1

    def check(self, y, a, wl, direct=False, gain=1.0, key="", label=""):
        """Sample by sample against float64 at window start a (times the float32 gain of the pool), and as a whole for
        crops of at least one block: relative RMS against the crop's RMS, or, for a quiet crop (RMS under 2^-6 of its
        rounding scale's: quiet graded blocks next to loud ones), against the scale's RMS.  Such a crop carries the
        rounding of its loud neighbours' transforms, which its own RMS does not measure - e.g. the direct stem of the
        aligned pool's candidate 0 at 42001 + 12293 samples: RMS 6.8e-4 of its scale's, error 1.3e-4 of its RMS and
        8.6e-8 of the scale's."""
        h = direct_path_rirs(self.h, TAPS) if direct else self.h
        y64, scale = render_check_inputs(self.x, h if self.P > 1 else h[0], self.mode, bounds=self.b, window=(a, wl))
        g = float(np.float32(gain))
        y64, scale = y64 * g, scale * g
        key = key + (" direct" if direct else "")
        quiet = wl >= B and _rms(y64) < _rms(scale) / 64
        worst, gl = check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL if wl >= B and not quiet else np.inf, n0=a,
                                 label=label)
        if quiet:
            gl = _rms(np.asarray(y, np.float64) - y64) / _rms(scale)
            assert gl <= TAU_GLOBAL, "%s: quiet crop, global RMS %.3g of the scale's > %.3g" % (label, gl, TAU_GLOBAL)
            with _STATS_LOCK:
                QUIET.setdefault(key, []).append(label)
        _note(key, worst, gl if wl >= B else 0.0)


def _bounds_of(idx, P):
    return np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)


def _random_cuts(rng, P, N, span=None):
    """Random cuts over [0, N], or over a random stretch of `span` samples (short segments: grid blocking)."""
    at = 0 if span is None else int(rng.integers(0, N - span))
    cuts = at + np.sort(rng.integers(0, (N if span is None else span) + 1, P - 2))
    return np.concatenate([[0], cuts, [N]]).astype(np.int32)

A_LENS = [64000, 3 * B + 5, 3001]


def a_aligned(rng):
    out = []
    for j, N in enumerate((65001, 90002, 130003)):
        P = 4 + j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        assert _choice(b, N, P, 4096) == 1
        out.append(ScaleCand(graded_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    return out


def a_mixed_k(rng):
    out = []
    for j, (N, L) in enumerate(((70001, 3000), (81002, 4097), (66003, 9000), (90000, 16384))):
        P = 3 + j % 3
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        out.append(ScaleCand(graded_dry(rng, N), delay_rirs(rng, P, 1, L)[0], b))
    return out


def a_static(rng):
    return [ScaleCand(graded_dry(rng, N), so.synth_rirs(rng, 1, 5, L), None)
            for N, L in ((66001, 2048), (70002, 4096), (80003, 3000))]

WB = 1024                      # window of the beacon draws

LB = 64                        # RIR taps of the beacon candidates

EDGE, Z0, Z1 = 3000, 10000, 20000

NS, NL, NN = 36000, 44000, 32000

SIL0 = Z0 + LB                 # crops [s, s + WB) with SIL0 <= s <= Z1 - WB render only the zone's zeros

SIL_SPAN = Z1 - WB - SIL0 + 1

PASS0, PASS_SPAN = EDGE + 100, Z0 - WB - EDGE - 200     # loud for every candidate

TSTARS = [0, 1, 30, 31, 32, 33, 63, 64]

SPECIAL = [0.0, -0.25, NAN, 1.0 - 2.0 ** -53, 1.0]       # tries 32.. of a special case: start 0 (3) and M - 1 (2)

LARGE = [(16, [0, 1, 2, 3, 4, 5, 6, 7], 0, 0),            # victim speaker 0 at lane 0, the shortest
         (16, [8, 9, 10, 11, 12, 13, 14, 15], 7, 15),     # victim speaker 7 at lane 15, the shortest
         (16, [0, 1, 2, 3, 4, 5, 6, 7], 7, 15),           # the shortest a noise reader at lane 15
         (16, [15, 14, 13, 12, 11, 10, 9, 8], 0, 0),      # speaker 0 at lane 15; the shortest a noise reader at lane 0
         (16, [3, 9, 12, 0, 6, 15, 1, 10], 7, 10),        # scattered speakers, the victim the shortest at lane 10
         (9, [1, 3, 5, 7, 8], 4, 8),
         (12, [11, 0, 4, 7], 0, 3),
         (16, [0, 1, 2, 3, 4, 5, 6, 7], 3, None)]

SMALL = [(1, [0], 0, 0),
         (3, [0, 1], 1, None),
         (3, [2, 0], 0, 2),
         (2, [1, 0], 1, 1),
         (3, [0, 1], 0, 2),
         (3, [1, 2], 1, 0)]


class Case:
    """One designed draw: `lanes` (pool, candidate) per reader, `speakers` reader lanes in speaker order, `u`, and the
    designed (start, used)."""

    def __init__(self, layout, tries, tstar, special, seed):
        nr, spk, victim, short = layout
        self.layout, self.tries, self.tstar = layout, tries, tstar
        self.speakers = list(spk)
        self.lanes = []
        for lane in range(nr):
            s = lane == short
            if lane in spk:
                zoned = spk.index(lane) == victim
                self.lanes.append(("spk", {(True, True): 0, (False, True): 1, (True, False): 2, (False, False): 3}[
                    (zoned, s)]))
            else:
                self.lanes.append(("noi", 1 if s else 0))
        self.bad_pick = None
        self._design(special, seed, victim_shortest=short is not None and short == spk[victim])

    def _design(self, special, seed, victim_shortest):
        rng = np.random.default_rng(seed)
        self.M = M = min(NS if p == "spk" and i < 2 else NN if p == "noi" and i == 1 else NL
                         for p, i in self.lanes) - WB + 1
        u = rng.random(self.tries)                               # tries after the kept one are never evaluated
        last = self.tries if self.tstar is None else self.tstar
        for t in range(last):
            u[t] = (SIL0 + (t * 7919 + seed) % SIL_SPAN + 0.5) / M
        if self.tstar is not None:
            u[self.tstar] = (PASS0 + (seed * 131) % PASS_SPAN + 0.5) / M
        if special:
            vals = SPECIAL if victim_shortest else SPECIAL[:3]  # M - 1 is silent only in the shortest's end zone
            for k, v in enumerate(vals):
                assert 32 + k < min(last, self.tries - 1)
                u[32 + k] = v
        self.u = u
        k = self.tries - 1 if self.tstar is None else self.tstar
        self.start, self.used = dr.start_of(u[k], M), (0 if self.tstar is None else self.tstar + 1)

STATS = {}                       # section / variant -> [worst local ratio, worst global relative RMS]

QUIET = {}                       # section / variant -> labels of crops whose global error is taken against the scale


_STATS_LOCK = threading.Lock()


def _note(key, worst, g):
    with _STATS_LOCK:                                    # (checks run on a thread pool)
        s = STATS.setdefault(key, [0.0, 0.0])
        s[0], s[1] = max(s[0], worst), max(s[1], g)


class NCand:
    """A candidate's whole normalised stems (what check_snap and the draw reference read as `full`)."""

    def __init__(self, c, full, full_d, loud):
        self.c, self.N, self.full, self.full_d, self.loud = c, c.N, full, full_d, loud


def normalised(R, render, c, target, taps=0):
    """render_host of the candidate alone with its target: (stem, direct stem or None, (LUFS, gain))."""
    lo = []
    d = [np.empty((c.C, c.N), np.float32)] if taps else None
    out = R.render_host([host_src(render, c, taps)], lufs_targets=[target], loudness_out=lo, sr=RATE, direct_outs=d)[0]
    return torch.from_numpy(out).cuda(), (torch.from_numpy(d[0]).cuda() if taps else None), lo[0]


# ------------------------------------------------------------------- host and tap-form pools at training scale
def report(title):
    """The worst float64 ratios of every section / variant key that starts with the title's section."""
    print("\n%s:" % title)
    for k in sorted(STATS):
        if k.startswith(title.split(":")[0]):
            print("  %-40s worst per-sample ratio %.3g, worst global relative RMS %.3g; %d quiet crops%s" % (
                k, *STATS[k], len(QUIET.get(k, [])), (" (first: %s)" % QUIET[k][0]) if k in QUIET else ""))


def pool_variant(cands):
    """The render kernel every slot of a pool of these candidates runs: static pools k_render_fast, pools of K > 1
    k_render<1,0>, moving pools whose every candidate picks aligned blocking on its own k_render_fast, and every other
    moving pool (mixed blocking renders on the grid) k_render<0,0>."""
    if cands[0].P == 1:
        return "k_render_fast static"
    if max(c.K for c in cands) > 1:
        return "k_render<1,0>"
    return "k_render_fast" if all(_choice(c.b, c.N, c.P, c.L) for c in cands) else "k_render<0,0>"


def normalised_cand(c):
    """The candidate with its RIR set divided by its abs-max in float32 (SS_RIR_NORMALIZE): the float64 reference of a
    slot of a normalised bank."""
    return ScaleCand(c.x, normalized(c.h), c.b)


class Pools:
    """One set of candidates as a device pool (key False) and as host pools of the bank forms in `form`: spectral banks
    (key True) and tap-form banks (key "taps"); banks shared between candidates when `share` names the RIR set of each,
    with direct sets of TAPS taps when `taps`, normalised when `normalize`, level tables and loudness targets.  `arms`
    lists the keys, the device pool's first; `refs` the candidates the float64 reference renders (normalised RIRs when
    `normalize`).  Counts the pinned bytes it holds."""

    def __init__(self, cands, taps=False, levels=None, lufs=None, share=None, host_only=False, form=("spectra",),
                 normalize=False):
        render, R = _R()
        self.cands, self.taps = cands, taps
        self.refs = [normalised_cand(c) for c in cands] if normalize else cands
        self.pools, self.banks = {}, []
        sets = share if share is not None else list(range(len(cands)))
        forms = (form,) if isinstance(form, str) else tuple(form)
        arms = ([] if host_only else [(False, False, "spectra")]) + [(f == "spectra" or f, True, f) for f in forms]
        for key, host, f in arms:
            banks = {}
            for c, r in zip(cands, sets):
                if r not in banks:
                    banks[r] = R.rir_bank(c.h if c.P > 1 else c.h[0], normalize, TAPS if taps else 0, host=host,
                                          form=f)
            self.banks += list(banks.values())
            srcs = []
            for c, r in zip(cands, sets):
                if c.P == 1:
                    srcs.append(render.StaticSource(c.x if host else to(c.x), banks[r]))
                elif host:
                    srcs.append(render.MovingSource(c.x, banks[r], c.b))
                else:
                    srcs.append(render.MovingSource(to(c.x), banks[r], to(c.b), bounds_host=c.b))
            self.pools[key] = R.source_pool(srcs, levels=levels, lufs_targets=lufs, sr=RATE)
        self.variant = pool_variant(cands)
        self.arms = list(self.pools)
        hosts = [k for k in self.arms if k is not False]
        self.pinned = sum(k.host_nbytes for k in self.banks) + sum(self.pools[k].host_nbytes for k in hosts)
        self.host = self.pools[hosts[-1]]                        # the arm the float64 checks read
        self.gains = self.host.loudness[:, 1]

    def gain(self, i):
        g = self.gains[i]
        return 1.0 if np.isnan(g) else float(g)

    def close(self):
        for p in self.pools.values():
            p.close()
        for k in self.banks:
            k.close()


def _hold(*pools):
    """The pinned host bytes the test's banks and pools hold, as the library counts them (host_nbytes; the renderer's own
    host staging buffers not included), printed and kept under 2 GB."""
    total = sum(p.pinned for p in pools)
    print("\npinned host memory of the banks and pools held (host_nbytes): %.1f MB" % (total / 1e6))
    assert total <= PINNED_MAX, total
    return total


def a_grid(rng):
    """Moving candidates with 59 segments of 0.3 to 3.8 k samples (grid blocking), pure-delay RIRs, graded dry
    signals."""
    out = []
    for j, N in enumerate((70001, 83002)):
        P = 60
        np.random.seed(500 + j)
        b = _bounds_of(so.setup_dynamic_interp(so.synth_path(rng, P), N)[0], P)
        assert _choice(b, N, P, 4096) == 0
        out.append(ScaleCand(graded_dry(rng, N), delay_rirs(rng, P, 3, 4096)[0], b))
    return out


def probe_starts(c, wl, rng):
    """0 and N - len; the maximisers of stage_cap, (K + 2) 4096 and b[s + 1] - 1 + (K + 2) 4096; starts where xa clamps
    to 0 and where xb clamps to N; starts with ws % 4 in {1, 2, 3}; all inside [0, N - len]."""
    last = c.N - wl
    d0 = (c.K + 2) * B
    s = {0, last, d0, d0 - 1, 1, last - 1, max(0, c.N - wl - 2 * B + 1)}
    for q in ([] if c.b is None else c.b[1:-1]):
        s.add(int(q) - 1 + d0)
    for m in (1, 2, 3):
        v = int(rng.integers(0, last + 1))
        s.add(v - v % 4 + m)
    return sorted(v for v in s if 0 <= v <= last)


def read_set(c, ws, wl, sets):
    """(bytes k_stage copies - whole float4s of dry samples and the rows of every set -, rows, dry samples)."""
    xa, xb, _, rows = (int(v[0]) for v in stage_set_np(c.N, c.P, c.C, c.K, c.b, [ws], wl))
    return 4 * (((xb + 3) & ~3) - (xa & ~3)) + sets * rows * B * 8, rows, xb - xa


class Probes:
    """A plan over every pool (arm) of `pl`: for every window length, `k` slots with device starts and one with a fixed
    start, all over the same pick and start tensors, NaN-filled guarded outputs."""

    def __init__(self, pl, lens, k, fixed):
        render, R = _R()
        self.pl, self.lens, self.k = pl, lens, k
        n = len(lens) * (k + 1)
        self.picks = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.starts = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.slots = []                               # (wl, fixed start or None)
        for wl, f in zip(lens, fixed):
            self.slots += [(wl, None)] * k + [(wl, f)]
        C = pl.cands[0].C
        self.plans, self.outs, self.douts = {}, {}, {}
        for arm, pool in pl.pools.items():
            srcs = [render.Pooled(pool, self.picks[j], (self.starts[j] if f is None else f, wl), TAPS if pl.taps else 0)
                    for j, (wl, f) in enumerate(self.slots)]
            self.outs[arm] = [Out(C, wl) for wl, _ in self.slots]
            self.douts[arm] = [Out(C, wl) for wl, _ in self.slots] if pl.taps else []
            self.plans[arm] = R.plan_device(srcs, [o.view() for o in self.outs[arm]],
                                            direct_outs=[o.view() for o in self.douts[arm]] if pl.taps else None)

    def run(self, pk, st):
        self.pk, self.st = list(pk), [s if f is None else f for s, (_, f) in zip(st, self.slots)]
        self.picks.copy_(torch.tensor(self.pk, dtype=torch.int32))
        self.starts.copy_(torch.tensor(st, dtype=torch.int32))
        R = _R()[1]
        self.launches, self.errors = {}, {}
        for arm in self.plans:
            for o in self.outs[arm] + self.douts[arm]:
                o.reset()
            R.reset_stats()
            self.plans[arm].run()
            self.launches[arm] = R.launch_count()
            self.errors[arm] = _device_errors(R)
        torch.cuda.synchronize()
        first = self.pl.arms[0]
        for arm in self.pl.arms[1:]:                      # (i) bit for bit the first arm's plan
            assert self.errors[arm] == self.errors[first], (arm, self.errors)
            for j in range(len(self.slots)):
                a, b = self.outs[first][j].get(), self.outs[arm][j].get()
                assert np.array_equal(a, b), ("twin", arm, j, self.pk[j], self.st[j])
                if self.pl.taps:
                    assert np.array_equal(self.douts[first][j].get(), self.douts[arm][j].get()), ("direct twin", arm, j)

    def check(self, key, label):
        last, jobs = self.pl.arms[-1], []
        for j, (wl, _) in enumerate(self.slots):          # (ii) float64, on a thread pool
            c = self.pl.refs[self.pk[j]]
            g = self.pl.gain(self.pk[j])
            what = "%s slot %d cand %d start %d len %d" % (label, j, self.pk[j], self.st[j], wl)
            jobs.append((c, self.outs[last][j].get(), self.st[j], wl, False, g, what))
            if self.pl.taps:
                jobs.append((c, self.douts[last][j].get(), self.st[j], wl, True, g, what + " direct"))
        pmap(lambda t: t[0].check(t[1], t[2], t[3], direct=t[4], gain=t[5], key=key, label=t[6]), jobs)

    def close(self):
        for p in self.plans.values():
            p.close()


def b_configs1(rng):
    """bench.make_inputs(16, 0): 32 configs[1] speakers (P = 40, C = 6, 30 s; every other dry signal gappy) and 16
    static 6-channel noises."""
    import bench
    items = bench.make_inputs(16, 0)
    spk = [ScaleCand(gappy_dry(rng, len(x)) if j % 2 else x, h, b) for j, (x, h, b) in enumerate(items)]
    N, C = bench.CFG["N"], bench.CFG["C"]
    noi = [ScaleCand((rng.standard_normal(N) * 0.05).astype(np.float32),
                (rng.standard_normal((1, C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32), None)
           for _ in range(16)]
    return spk, noi


class Training:
    """16 scenes: `layout` a list of (pools key, taps) per scene, the first two the mixture's speakers and the draw's,
    the rest its noises; one start per scene drawn by a 101-try CropDraw over mono level tables; one mono Mixture.  One
    plan per arm of the pools (Pools.arms, the same in every pool)."""

    def __init__(self, pools, layout, U=16):
        render, R = _R()
        self.pools, self.layout, self.U = pools, layout, U
        S = len(layout)
        self.picks = torch.zeros((U, S), dtype=torch.int32, device="cuda")
        self.starts = torch.zeros(U, dtype=torch.int32, device="cuda")
        self.u = torch.zeros((U, TRIES), dtype=torch.float64, device="cuda")
        self.used = torch.zeros(U, dtype=torch.int32, device="cuda")
        self.sirs = torch.zeros((U, 1), device="cuda")
        self.snr = torch.zeros(U, device="cuda")
        self.T = 4 * RATE
        self.plans, self.o = {}, {}
        self.arms = next(iter(pools.values())).arms
        for arm in self.arms:
            srcs, outs, douts, mixes, draws = [], [], [], [], []
            o = dict(outs=[], douts=[], mix=[], spk=[], rms=[])
            for u in range(U):
                base = len(srcs)
                for k, (key, taps) in enumerate(layout):
                    pl = pools[key]
                    srcs.append(render.Pooled(pl.pools[arm], self.picks[u, k], (self.starts[u], self.T),
                                              TAPS if taps else 0))
                    o["outs"].append(Out(pl.cands[0].C, self.T))
                    o["douts"].append(Out(pl.cands[0].C, self.T) if taps else None)
                o["mix"].append(Out(1, self.T))
                o["spk"].append(Out(2, self.T))
                o["rms"].append(Out(1, 2))
                mixes.append(render.Mixture([base, base + 1], list(range(base + 2, base + S)), self.sirs[u],
                                            self.snr[u], o["mix"][-1].view(self.T), o["spk"][-1].view(2, self.T),
                                            o["rms"][-1].view(2), mono=True))
                draws.append(render.CropDraw(self.starts[u], [base, base + 1], self.u[u], self.used[u]))
            self.o[arm] = o
            self.plans[arm] = R.plan_device(srcs, [x.view() for x in o["outs"]],
                                             direct_outs=[None if x is None else x.view() for x in o["douts"]],
                                             mixtures=mixes, draws=draws)

    def bufs(self, arm):
        o = self.o[arm]
        return o["outs"] + [x for x in o["douts"] if x is not None] + o["mix"] + o["spk"] + o["rms"]

    def draw(self, gen):
        for k, (key, _) in enumerate(self.layout):
            n = self.pools[key].host.n
            self.picks[:, k].copy_(torch.randint(0, n, (self.U,), generator=gen, device="cuda", dtype=torch.int32))
        self.u.uniform_(generator=gen)
        self.sirs.uniform_(-6, 6, generator=gen)
        self.snr.uniform_(10, 20, generator=gen)

    def run(self, gen, tables, run, full_check, what):
        """One run of every arm's plan; returns the number of draws checked against draw_reference."""
        self.draw(gen)
        R = _R()[1]
        drawn, self.launches = {}, {}
        for arm in self.arms:
            for x in self.bufs(arm):
                x.reset()
            self.starts.fill_(-1)
            self.used.fill_(-7)
            R.reset_stats()
            self.plans[arm].run()
            self.launches[arm] = R.launch_count()
            drawn[arm] = (self.starts.clone(), self.used.clone(), _device_errors(R))
        torch.cuda.synchronize()
        first = self.arms[0]
        for arm in self.arms[1:]:                                        # (i)
            for a, b in zip(self.bufs(first), self.bufs(arm)):
                assert np.array_equal(a.get(), b.get()), (what, arm)
            assert torch.equal(drawn[arm][0], drawn[first][0]) and torch.equal(drawn[arm][1], drawn[first][1]), arm
            assert drawn[arm][2] == drawn[first][2] == 0, (arm, drawn[arm][2], drawn[first][2])
        pk, st = self.picks.cpu().numpy(), self.starts.cpu().numpy()
        used, u = self.used.cpu().numpy(), self.u.cpu().numpy()
        sirs, snr = self.sirs.cpu().numpy(), self.snr.cpu().numpy()
        o, S, checked = self.o[self.arms[-1]], len(self.layout), 0
        for e in range(self.U):
            a = int(st[e])
            stems = []
            for k, (key, taps) in enumerate(self.layout):
                pl = self.pools[key]
                i = int(pk[e, k])
                y = o["outs"][S * e + k].get()
                stems.append(y)
                if full_check or e in (0, 7, 15):                       # (ii)
                    c = pl.refs[i]
                    label = "%s run %d scene %d stem %d cand %d start %d" % (what, run, e, k, i, a)
                    c.check(y, a, self.T, gain=pl.gain(i), key="B %s %s" % (what, pl.variant), label=label)
                    if taps:
                        c.check(o["douts"][S * e + k].get(), a, self.T, direct=True, gain=pl.gain(i),
                                key="B %s %s" % (what, pl.variant), label=label + " direct")
            check_mixture(np.stack([fold(s) for s in stems[:2]]), np.stack([fold(s) for s in stems[2:]]), sirs[e],
                          snr[e], o["mix"][e].get().reshape(-1), o["spk"][e].get().reshape(2, -1),
                          o["rms"][e].get().reshape(-1), "%s run %d scene %d" % (what, run, e))
            tabs = [tables[self.layout[k][0]][int(pk[e, k])] for k in range(2)]
            Nr = [self.pools[key].cands[int(pk[e, k])].N for k, (key, _) in enumerate(self.layout)]
            if dr.margins(tabs, [self.T, self.T], Nr, self.T, u[e]) < NEAR_DB:
                continue
            assert (a, int(used[e])) == dr.draw(tabs, [self.T, self.T], Nr, self.T, u[e]), (what, run, e)
            checked += 1
        return checked

    def close(self):
        for p in self.plans.values():
            p.close()


def _tables(pl):
    return [pl.host.level_table(i).cpu().numpy() for i in range(pl.host.n)]


def _training(pools, layout, what, runs=3, min_draws=30):
    R = _R()[1]
    tr = Training(pools, layout)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(77)
    tables = {k: _tables(p) for k, p in pools.items() if p.host.levels is not None}
    for k, p in pools.items():
        if p.host.levels is not None:
            for i in range(p.host.n):
                for arm in p.arms:
                    assert torch.equal(p.host.level_table(i), p.pools[arm].level_table(i)), (what, k, arm, i)
    try:
        R.check_device_errors()
        checked = sum(tr.run(gen, tables, r, r == 0, what) for r in range(runs))
        assert checked >= min_draws, checked
        for p in tr.plans.values():
            assert p.is_graph()
        R.check_device_errors()
        print("\n%s: %d draws checked against draw_reference; launches per run %s" % (what, checked, tr.launches))
        return tr.launches
    finally:
        tr.close()


def copy_batches(C, cands, first, form="spectra"):
    """render_host_stems' batching restated: candidate i's copy is its reverberant spectra (its taps, half the bytes,
    for a tap-form pool) and dry signal, each 256-aligned (stem_copy_bytes); the buffer holds max(largest copy, min(all copies, 256 MiB)) (stem_copy_cap); inside
    every stem group a batch takes candidates while they fit, and always at least one.  Returns every batch's first
    candidate."""
    row = 4 * B if form == "taps" else 8 * B
    cb = [align_up(row * c.P * C * c.K, 256) + align_up(4 * c.N, 256) for c in cands]
    cap = max(max(cb), min(sum(cb), STEM_BYTES))
    starts = []
    for g in range(len(first) - 1):
        lo = first[g]
        while lo < first[g + 1]:
            starts.append(lo)
            used, hi = 0, lo
            while hi < first[g + 1] and (hi == lo or used + cb[hi] <= cap):
                used += cb[hi]
                hi += 1
            lo = hi
    return starts, cap


def d_speakers(rng, L=4096):
    import bench
    items = bench.make_inputs(24, 0)
    N, P, C = 30 * RATE, 60, 6
    cut = {5: 1, 18: 7, 30: 13, 47: 29}
    out = []
    for j, (x, _, _) in enumerate(items):
        n = N - cut.get(j, 0)
        b = _random_cuts(rng, P, n)
        out.append(ScaleCand(gappy_dry(rng, n) * np.float32(4.0) if j % 2 else x[:n].copy(), so.synth_rirs(rng, P, C, L), b))
    return out


def d_giant(rng, P_giant=400):
    """A moving 8-channel pool: one candidate with P = P_giant and L = 12288 (315 MB of spectra at P = 400) between
    ordinary ones."""
    out = []
    for j in range(5):
        if j == 2:
            P, L, N = P_giant, 12288, 400003
        else:
            P, L, N = 5, 4096, 300001 + 7 * j
        out.append(ScaleCand(so.synth_dry(rng, N) * np.float32(0.5 + 0.25 * (j % 3)), so.synth_rirs(rng, P, 8, L),
                        np.round(np.linspace(0, N, P)).astype(np.int32)))
    return out


def host_alone(R, render, c, target):
    """render_host of the candidate alone over a device bank: the (C, N) stem and, with a target, (LUFS, gain)."""
    bank = R.rir_bank(c.h)
    try:
        lo = []
        y = R.render_host([render.MovingSource(c.x, bank, c.b)], lufs_targets=None if target is None else [target],
                          loudness_out=lo, sr=RATE)[0]
    finally:
        bank.close()
    return y, (tuple(lo[0]) if target is not None else None)


# ------------------------------------------------------------------- device pools and the dry beacon draws
class DevPool:
    """A device source pool over candidates (test_gpu_host_pool_scale.Cand), with direct sets of `taps` taps."""

    def __init__(self, cands, taps=0, levels=None):
        render, R = _R()
        self.cands, self.taps = cands, taps
        self.banks = [R.rir_bank(c.h if c.P > 1 else c.h[0], direct_taps=taps) for c in cands]
        self.srcs = [render.StaticSource(to(c.x), bk) if c.P == 1 else
                     render.MovingSource(to(c.x), bk, to(c.b), bounds_host=c.b) for c, bk in zip(cands, self.banks)]
        self.pool = R.source_pool(self.srcs, levels=levels)
        self.n_max = max(c.N for c in cands)
        # a K = 1 candidate of a pool whose candidates differ in K renders on the pool's blocking, not bit for bit as
        # alone (test_gpu_pool_lengths): its stems are held to float64 only
        self.bits = [c.K > 1 or all(o.K == 1 for o in cands) for c in cands]

    def ref(self, i, x, s, wl):
        """render_device of candidate i with dry x[:N] at the fixed window (s, wl): host (stem, direct stem or None)."""
        _, R = _R()
        c = self.cands[i]
        out = torch.empty((c.C, wl), device="cuda")
        dout = torch.empty((c.C, wl), device="cuda") if self.taps else None
        src = self.srcs[i] if x is None else self.srcs[i]._replace(dry=x[:c.N].contiguous())
        R.render_device([src._replace(window=(s, wl), direct_taps=self.taps)], [out],
                        direct_outs=[dout] if self.taps else None)
        return out.cpu().numpy(), (dout.cpu().numpy() if self.taps else None)

    def close(self):
        self.pool.close()
        for b in self.banks:
            b.close()



D_TRIES = [1, 2, 31, 32, 33, 101, 4096]



def dry_beacon(rng, N, zone_end):
    """A dry signal loud (about -4.4 dB) everywhere, and with `zone_end` silent on [0, EDGE), [Z0, Z1) and
    [zone_end - EDGE, zone_end): every crop inside a zone is exactly silent in the signal's own table."""
    x = so.synth_dry(rng, N) * np.float32(6.0)
    if zone_end:
        x[:EDGE] = 0.0
        x[Z0:Z1] = 0.0
        x[zone_end - EDGE:zone_end] = 0.0
    return x


def traj_beacon(rng, N):
    """A loud static 2-channel candidate with a 64-tap RIR (its pool's level table is loud everywhere)."""
    h = np.zeros((1, 2, 64), np.float32)
    h[0, :, 0] = 1.0
    h[0, :, 1:] = rng.standard_normal((2, 63)) * 0.05 * np.exp(-np.arange(1, 64) / 16.0)
    return ScaleCand(so.synth_dry(rng, N) * np.float32(6.0), h, None)



def d_combos():
    for tries in D_TRIES:
        for t in sorted({t for t in TSTARS if t < tries} | {tries - 1}) + [None]:
            yield tries, t


def d_cases(layouts, seeds=(0,)):
    out = []
    for seed in seeds:
        for n, (tries, t) in enumerate(d_combos()):
            for j, lay in enumerate(layouts):
                out.append(Case(lay, tries, t, False, 2000 + 1000 * seed + 17 * n + j))
                if tries > 37 and (t is None or t > 36) and seed == 0:
                    out.append(Case(lay, tries, t, True, 2000 + 1000 * seed + 17 * n + j + 7))
    return out


class DryDrawPlan:
    """A plan of the cases' draws: every speaker lane a dry-picked slot of the trajectory pool, except the loud speakers
    of every other draw with two or more, which are plain pooled slots (mixed); noise lanes slots of the noise pool.
    With `dp16` (a 16-bit pool of bw.dp's values) every other dry-picked lane, alternating by draw and lane, picks from
    it instead: a draw mixes 16-bit and float speakers, at every lane.  `lanes16` counts (draw, lane) of 16-bit picks."""

    def __init__(self, bw, cases, dp16=None):
        render, R = _R()
        self.cases = cases
        nd = len(cases)
        self.starts = torch.zeros(nd, dtype=torch.int32, device="cuda")
        self.used = torch.full((nd,), -7, dtype=torch.int32, device="cuda")
        self.u = torch.from_numpy(np.concatenate([c.u for c in cases])).cuda()
        pk, dk, self.what, self.slot0 = [], [], [], []
        for k, c in enumerate(cases):
            lanes = []
            victim = c.layout[2]
            for lane, (p, i) in enumerate(c.lanes):
                if p == "noi":
                    lanes.append(("noi", i))
                elif i in (1, 3) and k % 2 and c.speakers.index(lane) != victim:
                    lanes.append(("plain", 0 if i < 2 else 1))
                else:
                    lanes.append(("dry", i))
                pk.append(i if p == "noi" else (0 if i < 2 else 1))
                dk.append(i if p == "spk" else 0)
            self.what.append(lanes)
        self.picks = torch.tensor(pk, dtype=torch.int32, device="cuda")
        self.dpicks = torch.tensor(dk, dtype=torch.int32, device="cuda")
        self.out = torch.empty((len(pk), 2, WB), device="cuda")
        srcs, draws, off = [], [], 0
        self.lanes16 = []
        for k, c in enumerate(cases):
            base = len(srcs)
            self.slot0.append(base)
            for j, (p, _) in enumerate(self.what[k]):
                q = base + j
                pool = bw.np.pool if p == "noi" else bw.tp.pool
                dry = None
                if p == "dry":
                    i16 = dp16 is not None and (k + j) % 2 == 0
                    dry = render.DryPick(dp16 if i16 else bw.dp, self.dpicks[q])
                    if i16:
                        self.lanes16.append((k, j))
                srcs.append(render.Pooled(pool, self.picks[q], (self.starts[k], WB), 0, dry))
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
        worst = np.inf
        for k, c in enumerate(self.cases):
            label = (what, k, c.layout, c.tries, c.tstar)
            got = (int(starts[k]), int(used[k]))
            assert got == (c.start, c.used), (label, got, (c.start, c.used))
            lanes = self.what[k]
            tabs = [bw.Td[lanes[lane][1]] if lanes[lane][0] == "dry" else bw.Tp[lanes[lane][1]] for lane in c.speakers]
            Nr = [(bw.np if p == "noi" else bw.tp).cands[i if p == "noi" else (i if p == "plain" else int(i >= 2))].N
                  for p, i in lanes]
            D = [WB] * len(tabs)
            assert dr.draw(tabs, D, Nr, WB, c.u) == got, label
            m = dr.margins(tabs, D, Nr, WB, c.u)
            assert m >= 29.0, (label, m)                       # no draw near the threshold
            worst = min(worst, m)
            s = got[0]
            for j, x in enumerate(lanes):
                assert torch.equal(self.out[self.slot0[k] + j], bw.full[x][:, s:s + WB]), (label, j, x)
        return worst

    def close(self):
        self.plan.close()


