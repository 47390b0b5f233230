"""Candidates, pools, slots and training plans that the GPU pool and dry-pool tests build their worlds from.  Test
infrastructure."""
import ctypes

import numpy as np
import pytest
import torch

import draw_reference as dr
from direct_path import direct_path_rirs
from draw_reference import LEN, NEAR_DB, RATE, gappy_dry
from gpu_plumbing import _R, _rms, to
from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, delay_rirs, graded_dry, render_check_inputs
from window_cases import _choice

B = 4096
NAN = float("nan")


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


def _note(key, worst, g):
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
