"""Layout draws (ss_layout_draw; render.LayoutDraw) on the CPU, through k_layout's own code (ss_phases.cuh: the
Philox4x32-10 stream and layout_row, exported by tests/emu/ss_emu_layout.cu).
  - Philox4x32-10 gives Random123's known-answer vectors, and the uniform integers follow the stream word for word.
  - Emulated rows equal the Python restatement of tests/layout_reference.py entry for entry over many (seed, t, r),
    for streams and beds, and at the corpus edges: n = 1, every utterance longer than `total`, K exactly at the cap,
    rows cut at m = 1 and m = 128, beds whose end clip is dropped, selection by other lengths than the clips'.
  - The outcome frequencies match the host get_random_wav_path + _place_long_audio and get_random_wav_path_from_json +
    _place_background_audio loops within 5 standard errors, over the corpora of tests/test_dry_streams.py and
    tests/test_background_streams.py.
  - Every emulated row walks with no invalid entry (stream_entries, bg_entries).
  - render.LayoutDraw's structural refusals are ValueErrors raised before any tensor or C call.
The plan-level refusals and the kernel itself need a device: tests/test_gpu_layout_draw.py."""
import collections
import json
import random

import numpy as np
import pytest
import torch

import layout_reference as lr
from sonicsim_b200 import dry, render


@pytest.fixture(scope="module")
def emu():
    return lr.load_emu()


def rows(emu, seeds_ts, r, lengths, total, m, sample_rate, bed, select=None, K=None):
    """Emulated rows at each (seed, t) of seeds_ts: (ids, offsets, heads, counts) arrays of shape (rows, m)."""
    rng = np.ascontiguousarray(np.asarray(seeds_ts, dtype=np.int64).reshape(-1, 2))
    q = rng.shape[0]
    L = np.ascontiguousarray(lengths, dtype=np.int32)
    S = None if select is None else np.ascontiguousarray(select, dtype=np.int32)
    if K is None:
        K = (dry.background_audio_max_selected(L if S is None else S, total) if bed
             else dry.long_audio_max_selected(L, total))
    out = [np.zeros((q, m), np.int32) for _ in range(4)]
    emu.emu_layout_rows(rng.ctypes.data, q, r, L.ctypes.data, None if S is None else S.ctypes.data, L.size, m, total,
                        10 * sample_rate, K, out[0].ctypes.data, out[1].ctypes.data,
                        out[2].ctypes.data if bed else None, out[3].ctypes.data if bed else None)
    if not bed:
        out[2][:] = -1
        out[3][:] = -1
    return out


def walk(emu, row, lengths, bed):
    a = [np.ascontiguousarray(v, dtype=np.int32) for v in row]
    L = np.ascontiguousarray(lengths, dtype=np.int32)
    kept = np.zeros(1, np.int32)
    err = emu.emu_layout_walk(a[0].ctypes.data, a[1].ctypes.data, a[2].ctypes.data if bed else None,
                              a[3].ctypes.data if bed else None, a[0].size, L.ctypes.data, L.size, kept.ctypes.data)
    return int(kept[0]), err


def check_rows(emu, seeds_ts, r, lengths, total, m, sr, bed, select=None, K=None):
    """Emulated rows == the Python restatement, and every row walks clean; returns the restatement's notes."""
    got = rows(emu, seeds_ts, r, lengths, total, m, sr, bed, select, K)
    notes = collections.Counter()
    for q, (seed, t) in enumerate(seeds_ts):
        want, note = lr.layout_row(seed, t, r, list(lengths), total, m, sr, bed, None if select is None else list(select))
        row = [v[q].tolist() for v in got]
        assert row == want, (seed, t, r, row, want)
        kept, err = walk(emu, row, lengths, bed)
        assert err == 0 and kept == sum(1 for i in row[0] if i >= 0)
        assert lr.walk_rule(*row[:2], *(row[2:] if bed else (None, None)), lengths) == (kept, False)
        notes[note] += 1
        notes["entries"] += kept
        notes["full"] += kept == m
    return notes


def pairs(count, seed=0):
    g = np.random.default_rng(seed)
    s = g.integers(-2 ** 63, 2 ** 63 - 1, count, dtype=np.int64)
    t = g.integers(-2 ** 63, 2 ** 63 - 1, count, dtype=np.int64)
    t[: count // 2] = np.arange(count // 2)                # small counters too, as a training loop bumps them
    return list(zip(s.tolist(), t.tolist()))


# ------------------------------------------------------------------------------------------------- the generator
@pytest.mark.parametrize("ctr,key,want", [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_philox_known_answers(emu, ctr, key, want):
    c, k, out = np.array(ctr, np.uint32), np.array(key, np.uint32), np.zeros(4, np.uint32)
    emu.emu_philox(c.ctypes.data, k.ctypes.data, out.ctypes.data)
    assert out.tolist() == want
    assert lr.philox(ctr, key) == want


def test_uniform_integers_follow_the_stream(emu):
    g = np.random.default_rng(1)
    for seed, t in pairs(40, 1):
        r = int(g.integers(0, 1000))
        k = [1, 2, 3, 160001, 2 ** 31, 2 ** 32 + 5, 2 ** 63] + g.integers(1, 2 ** 40, 30).tolist()
        ks = np.array(k, np.uint64)
        out = np.zeros(len(k), np.uint64)
        emu.emu_rng_below(np.array([seed, t], np.int64).ctypes.data, r, ks.ctypes.data, len(k), out.ctypes.data)
        w = lr.Words(seed, t, r)
        assert out.tolist() == [w.below(v) for v in k]
        assert all(0 <= a < b for a, b in zip(out.tolist(), k))


# ---------------------------------------------------------------------------------------------- rows, entry for entry
@pytest.mark.parametrize("bed", [False, True])
def test_random_corpora_equal_the_restatement(emu, bed):
    g = np.random.default_rng(2 if bed else 3)
    for case in range(12):
        n = int(g.integers(1, 300))
        lengths = g.integers(1, 4000, n).tolist()
        total = int(g.integers(100, 30000))
        m = int(g.choice([1, 3, 16, 128]))
        sr = int(g.choice([1, 10, 100]))
        r = int(g.integers(0, 500))
        select = g.integers(0, 9000, n).tolist() if bed and case % 3 == 0 else None
        notes = check_rows(emu, pairs(60, case), r, lengths, total, m, sr, bed, select)
        assert notes["entries"] > 0


def test_n_of_one(emu):
    for bed in (False, True):
        notes = check_rows(emu, pairs(200, 4), 7, [500], 2000, 4, 10, bed)
        assert notes["entries"] > 100


def test_every_utterance_longer_than_total(emu):
    notes = check_rows(emu, pairs(100, 5), 0, [300, 400, 1000], 250, 8, 10, False)
    assert notes["entries"] == 0                      # nothing fits: every row is empty
    notes = check_rows(emu, pairs(100, 5), 0, [300, 400, 1000], 250, 8, 10, True)
    assert notes["entries"] + notes["dropped"] == 100   # a bed still takes the first clip as its end clip


def test_k_exactly_at_the_cap(emu):
    # streams: 1024 utterances of 10 fit in 10240 and no more; beds: 1023 clips of 1 stay below 0.4 * 2560
    assert dry.long_audio_max_selected([10] * 3000, 10240) == 1024
    notes = check_rows(emu, pairs(6, 6), 3, [10] * 3000, 10240, 128, 1, False)
    assert notes["full"] == 6                          # and the rows are cut at m = 128
    assert dry.background_audio_max_selected([1] * 2000, 2560) == 1024
    check_rows(emu, pairs(6, 7), 4, [1] * 2000, 2560, 128, 1, True)


def test_rows_cut_at_one_and_at_128(emu):
    lengths = [5] * 400 + [30] * 100
    for m in (1, 128):
        for bed in (False, True):
            notes = check_rows(emu, pairs(30, 8), 11, lengths, 6000 if not bed else 20000, m, 1, bed)
            assert notes["full"] > 0


def test_beds_whose_end_clip_is_dropped(emu):
    # short clips and tails of up to 200 samples: an end clip whose lead passes its samples is dropped
    notes = check_rows(emu, pairs(400, 9), 2, [3, 2, 4], 400, 8, 20, True)
    assert notes["dropped"] > 20 and notes[None] > 20


def test_select_lengths_quirk(emu):
    lens16 = [37, 61, 23, 90]
    sel = [(v * 441) // 160 for v in lens16]
    assert dry.background_audio_max_selected(sel, 150) == 1 and dry.background_audio_max_selected(lens16, 150) == 2
    check_rows(emu, pairs(300, 10), 5, lens16, 150, 8, 10, True, sel)


def test_same_counter_same_rows_and_the_next_counter_differs(emu):
    lengths = list(range(100, 400, 7))
    a = rows(emu, [(42, 9)] * 2, 0, lengths, 3000, 16, 10, False)
    assert np.array_equal(a[0][0], a[0][1]) and np.array_equal(a[1][0], a[1][1])
    b = rows(emu, [(42, 10), (42, 9)], 1, lengths, 3000, 16, 10, False)
    c = rows(emu, [(42, 9)], 1, lengths, 3000, 16, 10, False)
    assert not np.array_equal(a[1][0], b[1][0]) and not np.array_equal(b[1][0], c[1][0])   # t and r both move it


# ------------------------------------------------------------------------------------------------- distributions
def counts_of(table):
    return collections.Counter(table)


def assert_same_distribution(host, dev, R, min_keys):
    keys = set(host) | set(dev)
    assert len(keys) > min_keys
    for key in keys:
        p, q = host[key] / R, dev[key] / R
        sd = np.sqrt((p * (1 - p) + q * (1 - q)) / R)
        assert abs(p - q) <= 5 * sd + 1e-3, (key, p, q)


@pytest.mark.parametrize("m", [8, 2])
@pytest.mark.parametrize("lengths,total,sr", [([30, 40, 50], 120, 2), ([10, 25, 60, 5], 100, 1),
                                              ([7, 7, 20, 33, 41], 90, 1)])
def test_stream_frequencies_match_the_host_loop(emu, lengths, total, sr, m):
    R = 40000
    random.seed(1234)
    host = counts_of(lr.host_stream(lengths, total, sr)[:m] for _ in range(R))
    ids, offs, _, _ = rows(emu, [(77, t) for t in range(R)], 3, lengths, total, m, sr, False)
    dev = counts_of(tuple((i, o) for i, o in zip(ri, ro) if i >= 0) for ri, ro in zip(ids.tolist(), offs.tolist()))
    assert_same_distribution(host, dev, R, 20)


@pytest.mark.parametrize("different_select", [False, True])
def test_bed_frequencies_match_the_host_loop(emu, tmp_path, different_select):
    sr, total, R = 10, 150, 40000
    lens16 = [37, 61, 23, 90]
    sel = [(v * 441) // 160 for v in lens16] if different_select else lens16
    js = tmp_path / "bg.json"
    js.write_text(json.dumps({str(i): v for i, v in enumerate(sel)}))
    random.seed(5)
    host = counts_of(lr.host_bed(lens16, str(js), total, sr) for _ in range(R))
    lay = rows(emu, [(-3, t) for t in range(R)], 1, lens16, total, 8, sr, True, sel if different_select else None)
    dev = counts_of(tuple(e for e in zip(*[v[q].tolist() for v in lay]) if e[0] >= 0) for q in range(R))
    assert_same_distribution(host, dev, R, 20)


# ------------------------------------------------------------------------------------------------------ refusals
class _NoDevice:
    """A renderer stand-in: _device_layouts' structural checks run before any tensor check or C call."""
    device = 0


@pytest.mark.parametrize("why", ["not a draw", "slot out of range", "not a stream slot"])
def test_layout_draw_structural_refusals(why):
    stream = render.Pooled(None, None, (0, 10), dry=render.DryStream(None, None, None))
    plain = render.Pooled(None, None, (0, 10))
    rng = torch.zeros(2, dtype=torch.int64)
    sources = [stream, plain]
    layouts = {"not a draw": [(0, rng, 100)],
               "slot out of range": [render.LayoutDraw(2, rng, 100)],
               "not a stream slot": [render.LayoutDraw(1, rng, 100)]}[why]
    with pytest.raises(ValueError, match="layout"):
        render.Renderer._device_layouts(_NoDevice(), layouts, sources, ([], [None, None], None, None), [])


def test_layout_draw_fields():
    d = render.LayoutDraw(3, "rng", 960000)
    assert d.sample_rate == 16000 and d.select_lengths is None
    assert render.LayoutDraw._fields == ("slot", "rng", "total", "sample_rate", "select_lengths")
