"""The crop start loop of the separation dataloader (separation/look2hear/datas/movingdatamodule.py:81-99) restated over
float64 level tables, as ss_plan_draw defines it, and the level tables of ss_pool_levels in NumPy.  Test infrastructure.

The reference draws `start = random.randint(0, L - crop)` up to 101 times and rejects a start while any speaker's crop
has compute_mch_rms_dB (:29-32) below -40; after 101 rejections it keeps the last start.  Here randint(0, M - 1) is
M * u truncated, with u given, and a crop's mean square is (Q[s + len] - Q[s]) / D from the speaker's table.
tests/golden/crop_draw.npz pins this control flow to the unmodified reference lines."""
import math

import numpy as np
import torch

from oracle import sonicsim_oracle as so

NAN = float("nan")


def fold_mono(y):
    """The channel fold of the mixture kernels: float32 sum of the rows in channel order, then a division by C."""
    y = np.asarray(y, np.float32)
    v = y[0].copy()
    for c in range(1, y.shape[0]):
        v = (v + y[c]).astype(np.float32)
    return (v / np.float32(y.shape[0])).astype(np.float32)


def level_terms(y, mono):
    """e[n] of a (C, N) float32 stem: (double)(v * v) of the fold, or the float64 sum of the channels' float32 squares."""
    y = np.asarray(y, np.float32)
    if mono:
        v = fold_mono(y)
        return (v * v).astype(np.float64)
    e = np.zeros(y.shape[1], np.float64)
    for c in range(y.shape[0]):
        e += (y[c] * y[c]).astype(np.float64)
    return e


def level_table(y, mono, dtype=np.float64):
    """Q[0] = 0, Q[n + 1] = Q[n] + e[n] (sequential sums in `dtype`; np.longdouble gives a closer reference)."""
    e = level_terms(y, mono).astype(dtype)
    return np.concatenate([np.zeros(1, dtype), np.cumsum(e, dtype=dtype)])


def start_of(u, M):
    """Try start: min(floor(u * M), M - 1) in float64; u >= 1 gives M - 1, u < 0 or NaN gives 0."""
    v = math.floor(float(u) * float(M)) if np.isfinite(u) else (M - 1 if u > 0 else 0)
    if not v > 0:
        return 0
    return int(v) if v < M - 1 else M - 1


def level_db(Q, s, length, D):
    ms = (float(Q[s + length]) - float(Q[s])) / float(D)
    return 10.0 * math.log10(max(1e-20, ms))


def draw(tables, D, reader_N, length, u, threshold_db=-40.0):
    """(start, used) of one draw: `tables[k]`, `D[k]` the level table and crop element count of speaker k's picked
    candidate; `reader_N` the picked N of every reader (speakers and the rest).  Mirrors :81-99: for_idx counts the
    rejected tries, the loop ends after tries rejections with the last start."""
    M = min(int(n) for n in reader_N) - length + 1
    tries = len(u)
    start, for_idx = 0, 0
    while True:
        if for_idx > tries - 1:
            return start, 0
        start = start_of(u[for_idx], M)
        is_silence = 0
        for Q, d in zip(tables, D):
            if level_db(Q, start, length, d) < threshold_db:
                is_silence = 1
        if is_silence == 1:
            for_idx += 1
            continue
        return start, for_idx + 1


def margins(tables, D, reader_N, length, u, threshold_db=-40.0):
    """Least distance in dB, over the tries the draw evaluates (up to and including the kept one), between a speaker's
    level and the threshold: a draw whose margin is tiny may differ in the last bits of log10."""
    M = min(int(n) for n in reader_N) - length + 1
    start, used = draw(tables, D, reader_N, length, u, threshold_db)
    last = used if used > 0 else len(u)
    m = math.inf
    for t in range(last):
        s = start_of(u[t], M)
        for Q, d in zip(tables, D):
            m = min(m, abs(level_db(Q, s, length, d) - threshold_db))
    return m

TRIES = 101

TABLE_TOL = 1e-13              # |Q - Q_ref| <= TABLE_TOL * Q[N]: float64 scans of up to 4e5 non-negative terms

NEAR_DB = 1e-6                 # log10 of the device and of the host may differ in the last bit

RATE = 16000

LEN = 4 * RATE                 # the dataloader's 4 s crop


def gappy_dry(rng, N):
    """create_long_audio's layout: 0-10 s of silence, then a burst of speech (here 1-3 s of noise), and again."""
    x = np.zeros(N, np.float32)
    pos = int(rng.integers(0, 10 * RATE))
    while pos < N:
        n = int(rng.integers(RATE, 3 * RATE))
        k = min(n, N - pos)
        x[pos:pos + k] = so.synth_dry(rng, n)[:k]
        pos += n + int(rng.integers(0, 10 * RATE))
    return x


class Step:
    """B examples of two pooled speakers and one pooled noise sharing one start tensor, one mixture and one CropDraw
    each; NaN-filled outputs."""

    def __init__(self, R, render, spool, npool, B, thr=-40.0, tries=TRIES, draws=True, mono=True):
        dev = "cuda"
        self.B, self.thr, self.tries = B, thr, tries
        self.picks = torch.zeros((B, 3), dtype=torch.int32, device=dev)
        self.starts = torch.zeros(B, dtype=torch.int32, device=dev)
        self.u = torch.zeros((B, tries), dtype=torch.float64, device=dev)
        self.used = torch.full((B,), -7, dtype=torch.int32, device=dev)
        self.sirs = torch.zeros((B, 1), device=dev)
        self.snr = torch.full((B,), 15.0, device=dev)
        C = spool.C
        self.outs = [torch.empty((C, LEN), device=dev) for _ in range(3 * B)]
        self.mix = torch.empty((B, LEN) if mono else (B, C, LEN), device=dev)
        self.rms = torch.empty((B, 2), device=dev)
        self.srcs = []
        for b in range(B):
            self.srcs += [render.Pooled(spool, self.picks[b, 0], (self.starts[b], LEN)),
                          render.Pooled(spool, self.picks[b, 1], (self.starts[b], LEN)),
                          render.Pooled(npool, self.picks[b, 2], (self.starts[b], LEN))]
        self.mixtures = [render.Mixture([3 * b, 3 * b + 1], [3 * b + 2], self.sirs[b], self.snr[b], self.mix[b],
                                        rms_db=self.rms[b], mono=mono) for b in range(B)]
        self.draws = [render.CropDraw(self.starts[b], [3 * b, 3 * b + 1], self.u[b], self.used[b], thr)
                      for b in range(B)]
        self.plan = R.plan_device(self.srcs, self.outs, mixtures=self.mixtures, draws=self.draws if draws else None)

    def fill(self, gen, ns, nn):
        """New picks and u, drawn on the device (no host synchronisation); outputs NaN."""
        self.picks[:, :2].copy_(torch.randint(0, ns, (self.B, 2), generator=gen, device="cuda", dtype=torch.int32))
        self.picks[:, 2].copy_(torch.randint(0, nn, (self.B,), generator=gen, device="cuda", dtype=torch.int32))
        self.u.uniform_(generator=gen)
        for o in self.outs:
            o.fill_(NAN)
        self.rms.fill_(NAN)

    def snap(self):
        return dict(picks=self.picks.clone(), starts=self.starts.clone(), used=self.used.clone(), u=self.u.clone(),
                    outs=[o.clone() for o in self.outs], rms=self.rms.clone())


def check_snap(snap, spk, noi, Ts, D, thr, what):
    """Every example of one run against draw_reference on the device's tables; returns (checked, near) counts."""
    picks, starts = snap["picks"].cpu().numpy(), snap["starts"].cpu().numpy()
    used, u, rms = snap["used"].cpu().numpy(), snap["u"].cpu().numpy(), snap["rms"].cpu().numpy()
    checked = near = 0
    for b in range(len(starts)):
        p0, p1, pn = (int(v) for v in picks[b])
        Nr = [spk[p0].N, spk[p1].N, noi[pn].N]
        tabs = [Ts[p0], Ts[p1]]
        s, k = int(starts[b]), int(used[b])
        assert 0 <= s <= min(Nr) - LEN, (what, b, s, Nr)
        for j, c in enumerate((spk[p0], spk[p1], noi[pn])):
            assert torch.equal(snap["outs"][3 * b + j], c.full[:, s:s + LEN]), (what, b, j)
        if k > 0:
            assert rms[b].min() >= thr - 1e-5, (what, b, rms[b])
        if margins(tabs, [D, D], Nr, LEN, u[b], thr) < NEAR_DB:
            near += 1
            continue
        assert (s, k) == draw(tabs, [D, D], Nr, LEN, u[b], thr), (what, b, Nr)
        checked += 1
    return checked, near
