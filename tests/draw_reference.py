"""The crop start loop of the separation dataloader (separation/look2hear/datas/movingdatamodule.py:81-99) restated over
float64 level tables, as ss_plan_draw defines it, and the level tables of ss_pool_levels in NumPy.  Test infrastructure.

The reference draws `start = random.randint(0, L - crop)` up to 101 times and rejects a start while any speaker's crop
has compute_mch_rms_dB (:29-32) below -40; after 101 rejections it keeps the last start.  Here randint(0, M - 1) is
M * u truncated, with u given, and a crop's mean square is (Q[s + len] - Q[s]) / D from the speaker's table.
tests/golden/crop_draw.npz pins this control flow to the unmodified reference lines."""
import math

import numpy as np


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
