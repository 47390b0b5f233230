"""Dry streams (ss_dry_stream; render.DryStream, dry.long_audio_layouts) on the CPU.
  - The layout walk of ss_phases.cuh (stream_entries, exported by tests/emu/ss_emu_stream.cu) against the rule written
    out in Python: empty entries anywhere, each kind of invalid entry at the first, middle and last position, touching
    and 1-sample-overlapping placements, offsets at and beyond the stream's end, m = 1 and m = 128, 1-sample utterances.
  - k_stage's staging of a stream slot (stage_head, stream_resolve, stream_sample) gives the staged samples and view of
    a 16-bit dry pick of the explicitly assembled stream (k_stage<true>, tests/emu/ss_emu_compact.cu), bit for bit:
    placements at every residue mod 4 against the read set's ends, read sets that start inside a gap.
  - k_draw's stream draws (draw_silent_stream, per-utterance sums of the sparse tables) equal the float-table draws over
    the assembled stream's exact table, start for start and `used` for `used`: crops wholly in gaps, utterance
    boundaries at every residue mod 64 of either crop end, thresholds hit exactly.
  - dry.long_audio_layouts on CPU tensors: every row is a valid layout (ascending, without overlaps or repeats, gaps
    within 10 s, inside `total`), rows are cut at m; every row's selection, before placement drops entries, stops
    where get_random_wav_path stops (both stop conditions occur), with and without max_selected
    (long_audio_max_selected); and on pools of 3-5 utterances the frequency of every outcome matches the host
    get_random_wav_path + _place_long_audio loop, with and without max_selected and for m below the selection.
The refusals of render.DryStream and ss_plan_create_stream need a device context: tests/test_gpu_dry_streams.py."""
import collections
import ctypes
import random

import numpy as np
import pytest
import torch

from emu import build_emu
from sonicsim_b200 import dry, render

B = 4096
vp, i32, f32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float


@pytest.fixture(scope="module")
def emu():
    lib = build_emu.load("ss_emu_stream")
    lib.emu_stream_walk.argtypes = [vp, vp, i32, vp, i32, vp, vp, vp, vp]
    lib.emu_stream_stage.argtypes = [vp] + [i32] * 6 + [vp, vp, i32, vp, vp, i32, i32, vp, vp]
    lib.emu_draw_stream.argtypes = [vp, vp, i32, vp, vp, vp, i32, i32, i32, i32, vp, i32, f32, vp]
    return lib


@pytest.fixture(scope="module")
def compact():
    return build_emu.load("ss_emu_compact")


def walk_rule(ids, offsets, lengths):
    """The rule of include/sonicsim_b200.h in Python: (kept [(id, offset, len)], any invalid entry)."""
    kept, bad, end = [], False, 0
    for i, o in zip(ids, offsets):
        if i < 0:
            continue
        if i >= len(lengths) or o < 0 or o < end:
            bad = True
            continue
        kept.append((int(i), int(o), int(lengths[i])))
        end = o + lengths[i]
    return kept, bad


def assemble(ids, offsets, utts, cut):
    """The stream of `cut` samples a layout lays out: kept utterances in zeros, each cut at `cut`."""
    k = np.zeros(cut, np.int16)
    for i, o, n in walk_rule(ids, offsets, [u.size for u in utts])[0]:
        if o < cut:
            k[o:min(cut, o + n)] = utts[i][:min(n, cut - o)]
    return k


def squares(k):
    v = k.astype(np.float32) * np.float32(1.0 / 32768.0)
    return (v * v).astype(np.float64)


def full_table(k):
    return np.concatenate([[0.0], np.cumsum(squares(k))])


def sparse_table(Q):
    N = Q.size - 1
    return Q[np.minimum(np.arange(-(-N // 64) + 1) * 64, N)].copy()


def utterances(rng, n, lo, hi, amp=(0.01, 0.9)):
    return [np.clip(rng.standard_normal(int(rng.integers(lo, hi + 1))) * 32768 * rng.uniform(*amp), -32768,
                    32767).astype(np.int16) for _ in range(n)]


def arr(v):
    return np.ascontiguousarray(v, np.int32)


def call_walk(emu, ids, offsets, lengths):
    ids, offsets, lengths = arr(ids), arr(offsets), arr(lengths)
    m = ids.size
    kid, koff, klen = np.zeros(m, np.int32), np.zeros(m, np.int32), np.zeros(m, np.int32)
    cnt = ctypes.c_int()
    err = emu.emu_stream_walk(ids.ctypes.data, offsets.ctypes.data, m, lengths.ctypes.data, lengths.size,
                              kid.ctypes.data, koff.ctypes.data, klen.ctypes.data, ctypes.byref(cnt))
    k = cnt.value
    return list(zip(kid[:k].tolist(), koff[:k].tolist(), klen[:k].tolist())), err


# --------------------------------------------------------------------------------------------------------- the walk
def test_walk_examples(emu):
    L = [10, 1, 5, 7]
    cases = [
        # (ids, offsets, kept, invalid)
        ([0], [0], [(0, 0, 10)], False),
        ([-1, 0, -5], [99, 3, -7], [(0, 3, 10)], False),                   # empty entries skip whatever their offset
        ([0, 1], [0, 10], [(0, 0, 10), (1, 10, 1)], False),                # touching
        ([0, 1], [0, 9], [(0, 0, 10)], True),                              # a 1-sample overlap
        ([1, 1, 1], [0, 1, 2], [(1, 0, 1), (1, 1, 1), (1, 2, 1)], False),  # 1-sample utterances, touching, repeated
        ([4, 0], [0, 0], [(0, 0, 10)], True),                              # id == n
        ([0, 2, 3], [5, 3, 20], [(0, 5, 10), (3, 20, 7)], True),           # an offset before end, then valid again
        ([0, -1, 2], [0, 0, -1], [(0, 0, 10)], True),                      # a negative offset at the end
        ([2, 3], [1 << 30, (1 << 30) + 5], [(2, 1 << 30, 5), (3, (1 << 30) + 5, 7)], False),
        ([2, 3], [2147483647 - 3, 2147483647], [(2, 2147483647 - 3, 5)], True),   # the end beyond int32 still rules
    ]
    for ids, offs, kept, bad in cases:
        got, err = call_walk(emu, ids, offs, L)
        assert got == kept, (ids, offs)
        assert err == (32 if bad else 0), (ids, offs)
        assert walk_rule(ids, offs, L) == (kept, bad)


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("kind", ["id_n", "id_big", "negative", "overlap"])
def test_every_invalid_kind_at_every_position(emu, where, kind):
    L = [100] * 6
    ids, offs = [0, 1, 2, 3, 4], [0, 200, 400, 600, 800]
    j = {"first": 0, "middle": 2, "last": 4}[where]
    if kind == "id_n":
        ids[j] = 6
    elif kind == "id_big":
        ids[j] = 1 << 30
    elif kind == "negative":
        offs[j] = -1 if j == 0 else -(1 << 31)
    else:
        offs[j] = offs[j - 1] + 99 if j else 0
        if j == 0:                                      # the first entry cannot overlap: put one in front of it
            ids, offs = [5] + ids, [50] + offs
            j = 1
    got, err = call_walk(emu, ids, offs, L)
    kept, bad = walk_rule(ids, offs, L)
    assert bad and err == 32
    assert got == kept
    assert len(got) == len(ids) - 1                     # only the invalid entry is skipped


@pytest.mark.parametrize("m", [1, 2, 127, 128])
def test_random_layouts_follow_the_rule(emu, m):
    rng = np.random.default_rng(m)
    for _ in range(200):
        n = int(rng.integers(1, 9))
        L = rng.integers(1, 50, n).tolist()
        ids = rng.integers(-2, n + 2, m)
        offs = np.cumsum(rng.integers(-20, 60, m)) + int(rng.integers(-5, 5))
        got, err = call_walk(emu, ids, offs, L)
        kept, bad = walk_rule(ids.tolist(), offs.tolist(), L)
        assert got == kept and err == (32 if bad else 0)


# ------------------------------------------------------------------------------------------------------ the staging
def stage_stream(emu, bounds, N, P, K, ws, wl, ids, offs, utts, cut):
    ids, offs = arr(ids), arr(offs)
    lengths = arr([u.size for u in utts])
    sig = (ctypes.c_void_p * len(utts))(*[u.ctypes.data for u in utts])
    out = np.full(cut + 16, np.nan, np.float32)
    info = np.zeros(3, np.int32)
    err = emu.emu_stream_stage(bounds.ctypes.data, N, P, 2, K, ws, wl, ids.ctypes.data, offs.ctypes.data, ids.size,
                               lengths.ctypes.data, ctypes.cast(sig, ctypes.c_void_p), len(utts), cut, out.ctypes.data,
                               info.ctypes.data)
    return out[:info[1] - info[0]], info, err


def stage_pick(compact, bounds, N, P, K, ws, wl, k):
    """A 16-bit dry pick of the assembled stream k (k_stage<true>): its staged samples and [x0, x1)."""
    d = k.astype(np.float32) * np.float32(1.0 / 32768.0)
    of, oi = np.full(k.size + 16, np.nan, np.float32), np.full(k.size + 16, np.nan, np.float32)
    info = np.zeros(8, np.int32)
    compact.emu_stage_i16(bounds.ctypes.data, N, P, 2, K, ws, wl, d.ctypes.data, k.ctypes.data, k.size, 1, 0,
                          of.ctypes.data, oi.ctypes.data, info.ctypes.data)
    return oi[:info[3] - info[2]], info


def trajectory(rng, N, P):
    if P == 1:
        return np.zeros(1, np.int32)
    inner = np.sort(rng.choice(np.arange(1, N - 1), P - 2, replace=False)) if P > 2 else []
    return np.concatenate([[0], inner, [N]]).astype(np.int32)


@pytest.mark.parametrize("P,K", [(1, 1), (5, 2), (9, 3)])
def test_staged_samples_equal_the_assembled_pick(emu, compact, P, K):
    rng = np.random.default_rng(P + 10 * K)
    for trial in range(10):
        N = int(rng.integers(4 * B, 14 * B)) + int(rng.integers(0, 4))
        cut = N + int(rng.integers(0, 70))              # the pool's longest candidate: this one or a longer one
        utts = utterances(rng, 6, 1, 3 * B)
        bounds = trajectory(rng, N, P)
        wl = int(rng.integers(1, N // 2))
        for ws in sorted({0, N - wl, int(rng.integers(0, N - wl + 1)), min(N - wl, (K + 2) * B)}):
            x0 = max(0, ws - (K + 2) * B) & ~3
            x1 = (min(N, ws + wl + 2 * B) + 3) & ~3
            for r in range(8):
                # a placement whose start (r < 4) or end (r >= 4) sits at residue r % 4 after x0, one near x1, the rest
                # scattered; the read set then starts inside a gap or an utterance as the draw falls
                i0 = int(rng.integers(0, 6))
                a = x0 + 4 * int(rng.integers(0, 8)) + (r % 4) - (utts[i0].size if r >= 4 else 0)
                b = x1 - 4 * int(rng.integers(0, 8)) + (r % 4)
                cand = [(i0, a), (int(rng.integers(0, 6)), b)] + [
                    (int(rng.integers(0, 6)), int(rng.integers(0, cut))) for _ in range(int(rng.integers(0, 12)))]
                cand += [(-1, 0)] * int(rng.integers(0, 3))
                rng.shuffle(cand)
                cand.sort(key=lambda t: t[1])
                ids, offs = [c[0] for c in cand], [c[1] for c in cand]
                got, info, err = stage_stream(emu, bounds, N, P, K, ws, wl, ids, offs, utts, cut)
                kept, bad = walk_rule(ids, offs, [u.size for u in utts])
                assert err == (32 if bad else 0)
                assert info[2] == 1 and (info[0], info[1]) == (x0, x1)
                k = assemble(ids, offs, utts, cut)
                want, pinfo = stage_pick(compact, bounds, N, P, K, ws, wl, k)
                assert (pinfo[2], pinfo[3]) == (x0, x1)
                assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (trial, ws, r)


def test_read_set_inside_a_gap_stages_zeros(emu):
    N, K = 20 * B, 1
    utts = [np.full(100, 1000, np.int16), np.full(50, -7, np.int16)]
    ws, wl = 10 * B, B
    got, info, err = stage_stream(emu, np.zeros(1, np.int32), N, 1, K, ws, wl, [0, 1], [10, N - 60], utts, N)
    assert err == 0 and np.all(got == 0.0) and got.size == info[1] - info[0]


# ------------------------------------------------------------------------------------------------------- the draws
def draw_stream(emu, ids, offs, utts, cut, M, length, u, thr):
    ids, offs = arr(ids), arr(offs)
    lengths = arr([x.size for x in utts])
    qs = [sparse_table(full_table(x)) for x in utts]
    sig = (ctypes.c_void_p * len(utts))(*[x.ctypes.data for x in utts])
    lev = (ctypes.c_void_p * len(utts))(*[q.ctypes.data for q in qs])
    u = np.ascontiguousarray(u, np.float64)
    used = ctypes.c_int32()
    s = emu.emu_draw_stream(ids.ctypes.data, offs.ctypes.data, ids.size, lengths.ctypes.data,
                            ctypes.cast(sig, ctypes.c_void_p), ctypes.cast(lev, ctypes.c_void_p), len(utts), cut, M,
                            length, u.ctypes.data, u.size, float(thr), ctypes.byref(used))
    return s, used.value


def draw_table(compact, k, M, length, u, thr):
    """The float-table draw over the assembled stream's full table (D = len)."""
    Q = full_table(k)
    Qp = (ctypes.c_void_p * 1)(Q.ctypes.data)
    xp = (ctypes.c_void_p * 1)(None)
    D = np.full(1, float(length))
    u = np.ascontiguousarray(u, np.float64)
    used = ctypes.c_int32()
    s = compact.emu_draw_i16(ctypes.cast(Qp, ctypes.c_void_p), ctypes.cast(Qp, ctypes.c_void_p),
                             ctypes.cast(xp, ctypes.c_void_p), D.ctypes.data, 1, M, length, u.ctypes.data, u.size,
                             float(thr), ctypes.byref(used))
    return s, used.value


def test_draws_equal_the_assembled_table_draws(emu, compact):
    rng = np.random.default_rng(5)
    rejected = 0
    for trial in range(60):
        utts = utterances(rng, int(rng.integers(1, 7)), 1, 20000)
        N = int(rng.integers(20000, 90000))
        m = int(rng.integers(1, 20))
        ids = rng.integers(-1, len(utts) + 1, m).tolist()
        offs = np.sort(rng.integers(-10, N + 100, m)).tolist()
        length = int(rng.choice([1, 64, 1000, 4000, 16000]))
        M = N - length + 1
        u = rng.random(int(rng.integers(1, 200)))
        u[-1] = 1.0                                     # the last try ends at N
        k = assemble(ids, offs, utts, N)
        for thr in (-200.0, -60.0, -35.0, -20.0, 0.0):
            a, b = draw_stream(emu, ids, offs, utts, N, M, length, u, thr), draw_table(compact, k, M, length, u, thr)
            assert a == b, (trial, thr)
            rejected += a[1] != 1
    assert rejected > 30


def test_utterance_boundaries_at_every_residue_of_either_crop_end(emu, compact):
    rng = np.random.default_rng(11)
    utts = utterances(rng, 4, 200, 900)
    N, length = 8192, 333
    M = N - length + 1
    for r in range(64):
        for end in (0, 1):
            s0 = 1024 + r + 64 * int(rng.integers(0, 8))
            edge = s0 + (length if end else 0)          # an utterance starts or ends at either crop end
            ids = [0, 1, 2, 3]
            if r % 2:
                offs = [100, edge, edge + utts[1].size + 5, 7000]
            else:
                offs = [100, edge - utts[1].size, edge + 3, 7000]
            if offs[1] < 100 + utts[0].size:
                offs[1] = 100 + utts[0].size
            k = assemble(ids, offs, utts, N)
            u = [(s0 + 0.5) / M, (s0 + 1.5) / M, 0.25, 1.0]
            for thr in (-80.0, -30.0, -15.0, -5.0):
                assert draw_stream(emu, ids, offs, utts, N, M, length, u, thr) == \
                    draw_table(compact, k, M, length, u, thr), (r, end, thr)


def test_draw_thresholds_hit_exactly(emu, compact):
    N, length = 4096, 256
    utt = [np.full(2048, -32768, np.int16)]             # v = -1: ms = 1, 0 dB exactly; zeros: -200 dB
    ids, offs = [-1, 0], [5, 2048]
    k = assemble(ids, offs, utt, N)
    M = N - length + 1
    u_gap, u_loud, u_end = 0.0, 2048.5 / M, 1.0
    for u, thr, silent in [(u_gap, -200.0, False), (u_gap, -199.0, True), (u_loud, 0.0, False), (u_loud, 1e-3, True),
                           (u_end, 0.0, False), (u_end, 1e-3, True)]:
        a = draw_stream(emu, ids, offs, utt, N, M, length, [u], thr)
        assert a == draw_table(compact, k, M, length, [u], thr)
        assert a[1] == (0 if silent else 1), (u, thr)


# --------------------------------------------------------------------------------------------- long_audio_layouts
def host_layout(lengths, total, sample_rate):
    """get_random_wav_path's selection on lengths, then _place_long_audio: [(id, offset)] in stream order."""
    cands, chosen, acc = list(range(len(lengths))), [], 0
    while cands and acc < total * 0.9:
        pick = random.choice(cands)
        if acc + lengths[pick] > total:
            break
        chosen.append(pick)
        acc += lengths[pick]
        cands.remove(pick)
    places = dry._place_long_audio([lengths[c] for c in chosen], total, sample_rate)[0]
    return tuple((chosen[k], dst) for k, dst, _, _ in places)


def test_layout_rows_obey_the_rules():
    g = torch.Generator().manual_seed(3)
    sr, total, m = 100, 6000, 40
    lengths = torch.randint(50, 3500, (30,), generator=g)
    ids, offs = dry.long_audio_layouts(lengths, total, m, 500, generator=g, sample_rate=sr)
    assert ids.shape == offs.shape == (500, m) and ids.dtype == offs.dtype == torch.int32
    L = lengths.tolist()
    for row_i, row_o in zip(ids.tolist(), offs.tolist()):
        used = [(i, o) for i, o in zip(row_i, row_o) if i >= 0]
        assert all(i == -1 and o == -1 for i, o in zip(row_i[len(used):], row_o[len(used):]))
        assert len({i for i, _ in used}) == len(used)   # without replacement
        cur = 0
        for i, o in used:
            assert 0 <= o - cur <= 10 * sr             # the gap in front of it
            cur = o + L[i]
            assert cur <= total
        kept, bad = walk_rule(row_i, row_o, L)
        assert not bad and len(kept) == len(used)
        assert sum(L[i] for i, _ in used) <= total


@pytest.mark.parametrize("width", [None, "bound"])
def test_selection_stops_where_get_random_wav_path_stops(width):
    """The selection of every row, before placement drops entries: its chosen prefix is taken while the running total
    is below 0.9 * total and each taken utterance fits, and the first entry after it (if any) fails one of the two."""
    g = torch.Generator().manual_seed(4)
    total = 6000
    lengths = torch.randint(50, 3500, (40,), generator=g)
    w = lengths.numel() if width is None else dry.long_audio_max_selected(lengths, total)
    sel, chosen = dry._long_audio_selection(lengths, total, 400, w, {"generator": g, "device": lengths.device})
    assert sel.shape == chosen.shape == (400, w)
    L = lengths.tolist()
    stops = collections.Counter()
    for row, ch in zip(sel.tolist(), chosen.tolist()):
        assert len(set(row)) == len(row)                # a random order without replacement
        k = sum(ch)
        assert ch == [True] * k + [False] * (w - k)     # a prefix
        acc = 0
        for i in row[:k]:
            assert acc < 0.9 * total and acc + L[i] <= total
            acc += L[i]
        if k < w:
            nxt = L[row[k]]
            assert acc >= 0.9 * total or acc + nxt > total
            stops["threshold" if acc >= 0.9 * total else "overflow"] += 1
        else:
            assert k == len(L) or width is not None     # (a bounded width cannot cut a selection short:)
            if width is not None:
                assert acc + min(L[i] for i in set(range(len(L))) - set(row)) > total or k == len(L)
    assert stops["threshold"] > 20 and stops["overflow"] > 20   # both stop conditions occur


def test_max_selected_is_the_longest_possible_selection():
    assert dry.long_audio_max_selected([5, 1, 3, 10], 9) == 3          # 1 + 3 + 5
    assert dry.long_audio_max_selected(torch.tensor([5, 1, 3, 10]), 8) == 2
    assert dry.long_audio_max_selected([50, 60], 10) == 1              # at least 1
    assert dry.long_audio_max_selected([2, 2, 2], 100) == 3


def test_layouts_are_cut_at_m():
    g = torch.Generator().manual_seed(0)
    lengths = torch.full((50,), 10)
    ids, offs = dry.long_audio_layouts(lengths, 2000, 4, 20, generator=g, sample_rate=1)
    assert (ids >= 0).all() and ids.shape == (20, 4)    # every row would place more: its first 4 in stream order
    assert (offs[:, 1:] > offs[:, :-1]).all()


def test_layouts_need_no_host_sync_and_take_a_generator():
    lengths = torch.tensor([30, 40, 50])
    a = dry.long_audio_layouts(lengths, 120, 8, 16, generator=torch.Generator().manual_seed(9), sample_rate=2)
    b = dry.long_audio_layouts(lengths, 120, 8, 16, generator=torch.Generator().manual_seed(9), sample_rate=2)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    with pytest.raises(ValueError):
        dry.long_audio_layouts(lengths, 120, 129, 1)


@pytest.mark.parametrize("bounded", [False, True])
@pytest.mark.parametrize("m", [8, 2])
@pytest.mark.parametrize("lengths,total,sr", [([30, 40, 50], 120, 2), ([10, 25, 60, 5], 100, 1),
                                              ([7, 7, 20, 33, 41], 90, 1)])
def test_outcome_frequencies_match_the_host_loop(lengths, total, sr, m, bounded):
    """Every outcome (the placed (id, offset) sequence, its first m) at the host loop's frequency, with and without
    max_selected (the last pool's bound, 4, is below its n).  With R draws on each side, each frequency has a standard
    error of at most sqrt(p (1 - p) / R); the test allows 5 of them, combined over both sides, plus 1e-3, and requires
    outcomes the host never produced in R draws to stay as rare on the device side."""
    R = 40000
    random.seed(1234)
    host = collections.Counter(host_layout(lengths, total, sr)[:m] for _ in range(R))
    ids, offs = dry.long_audio_layouts(torch.tensor(lengths), total, m, R, generator=torch.Generator().manual_seed(5),
                                       sample_rate=sr,
                                       max_selected=dry.long_audio_max_selected(lengths, total) if bounded else None)
    dev = collections.Counter(tuple((i, o) for i, o in zip(ri, ro) if i >= 0)
                              for ri, ro in zip(ids.tolist(), offs.tolist()))
    for key in set(host) | set(dev):
        p, q = host[key] / R, dev[key] / R
        sd = np.sqrt((p * (1 - p) + q * (1 - q)) / R)
        assert abs(p - q) <= 5 * sd + 1e-3, (key, p, q)
    assert len(host) > 20                               # many distinct outcomes: gaps and orders vary


# ------------------------------------------------------------------------------------------------------- refusals
def test_dry_stream_is_a_named_tuple_of_three():
    d = render.DryStream("pool", "ids", "offsets")
    assert d.pool == "pool" and d.ids == "ids" and d.offsets == "offsets"
    assert render.DryStream._fields == ("pool", "ids", "offsets")
