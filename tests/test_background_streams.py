"""Background streams (ss_bg_stream; render.BackgroundStream, dry.background_audio_layouts, dry.background_clips) on the
CPU.
  - The layout walk of ss_phases.cuh (bg_entries, exported by tests/emu/ss_emu_background.cu) against the rule written
    out in Python: empty entries anywhere, each kind of invalid entry at the first, middle and last position, touching
    placements, heads and counts at the clip's edges, m = 1 and m = 128.
  - k_stage's staging of a bed slot (stage_head, bg_resolve, bg_sample) gives the assembled bed's samples, for int16 and
    float32 clips, with entries that reach or start past the cut, and the view of a dry-picked slot.
  - dry.background_audio_layouts: every row is a valid layout inside `total` with its selection stop; the outcome
    frequencies (clips per bed, an end clip or not, its lead, trail and count) match the host
    get_random_wav_path_from_json + _place_background_audio loop, also with select_lengths other than lengths.
  - dry.background_clips equals what create_background_audio adds, for 44.1 kHz stereo and 16 kHz mono clips.
The refusals of render.BackgroundStream and ss_plan_create_bg need a device context: tests/test_gpu_background_streams.py."""
import collections
import ctypes
import json
import random

import numpy as np
import pytest
import torch

from emu import build_emu
from sonicsim_b200 import dry

vp, i32 = ctypes.c_void_p, ctypes.c_int


@pytest.fixture(scope="module")
def emu():
    lib = build_emu.load("ss_emu_background")
    lib.emu_bg_walk.argtypes = [vp] * 4 + [i32, vp, i32] + [vp] * 5
    lib.emu_bg_stage.argtypes = [vp] + [i32] * 6 + [vp] * 4 + [i32, vp, vp, i32, i32, i32, vp, vp]
    return lib


def walk_rule(lay, lengths):
    """The rule of include/sonicsim_b200.h in Python: (kept [(id, offset, head, count)], any invalid entry)."""
    kept, bad, end = [], False, 0
    for i, o, h, c in zip(*lay):
        if i < 0:
            continue
        if i >= len(lengths) or o < 0 or h < 0 or c < 1 or h + c > lengths[i] or o < end:
            bad = True
            continue
        kept.append((int(i), int(o), int(h), int(c)))
        end = o + c
    return kept, bad


def arr(v):
    return np.ascontiguousarray(v, np.int32)


def call_walk(emu, lay, lengths):
    a = [arr(v) for v in lay]
    lengths = arr(lengths)
    m = a[0].size
    out = [np.zeros(m, np.int32) for _ in range(4)]
    cnt = ctypes.c_int()
    err = emu.emu_bg_walk(*[v.ctypes.data for v in a], m, lengths.ctypes.data, lengths.size,
                          *[v.ctypes.data for v in out], ctypes.byref(cnt))
    k = cnt.value
    return list(zip(*[v[:k].tolist() for v in out])), err


# --------------------------------------------------------------------------------------------------------- the walk
def test_walk_examples(emu):
    L = [10, 1, 5, 7]
    cases = [
        # (ids, offsets, heads, counts), kept, invalid
        (([0], [0], [0], [10]), [(0, 0, 0, 10)], False),
        (([-1, 0, -5], [99, 3, -7], [-4, 9, 0], [0, 1, 0]), [(0, 3, 9, 1)], False),   # empty entries skip anything
        (([0, 1], [0, 10], [2, 0], [8, 1]), [(0, 0, 2, 8), (1, 10, 0, 1)], False),    # touching
        (([0, 1], [0, 7], [2, 0], [8, 1]), [(0, 0, 2, 8)], True),                     # a 1-sample overlap
        (([0], [0], [9], [1]), [(0, 0, 9, 1)], False),                               # the clip's last sample
        (([0], [0], [9], [2]), [], True),                                            # one past the clip
        (([0], [0], [10], [1]), [], True),                                           # a head at the clip's end
        (([0], [0], [-1], [3]), [], True),
        (([0], [0], [0], [0]), [], True),
        (([4, 2], [0, 0], [0, 0], [1, 5]), [(2, 0, 0, 5)], True),                    # id == n
        (([2, 3], [2147483647 - 3, 2147483647], [0, 0], [4, 1]), [(2, 2147483647 - 3, 0, 4)], True),
    ]
    for lay, kept, bad in cases:
        got, err = call_walk(emu, lay, L)
        assert got == kept and bool(err) == bad and err in (0, 32), (lay, got, err)
        assert walk_rule(lay, L) == (kept, bad)


def test_walk_every_invalid_kind_at_every_position(emu):
    L = [30, 12, 1, 25]
    base = ([0, 1, 3, 2], [0, 30, 40, 60], [0, 2, 5, 0], [30, 10, 20, 1])        # touching placements
    assert walk_rule(base, L) == ([(0, 0, 0, 30), (1, 30, 2, 10), (3, 40, 5, 20), (2, 60, 0, 1)], False)
    kinds = [lambda e: (4, e[1], e[2], e[3]), lambda e: (e[0], -1, e[2], e[3]), lambda e: (e[0], e[1], -1, e[3]),
             lambda e: (e[0], e[1], e[2], 0), lambda e: (e[0], e[1], e[2], L[e[0]] - e[2] + 1),
             lambda e: (e[0], e[1] - 1, e[2], e[3])]
    for pos in range(4):
        for kind in kinds:
            lay = [list(v) for v in base]
            e = kind(tuple(v[pos] for v in lay))
            for q in range(4):
                lay[q][pos] = e[q]
            want = walk_rule(lay, L)
            assert want[1]
            assert call_walk(emu, lay, L) == (want[0], 32), (pos, e)


def test_walk_random_layouts(emu):
    rng = np.random.default_rng(4)
    L = list(rng.integers(1, 50, 9))
    for m in (1, 2, 7, 128):
        for _ in range(300):
            ids = rng.integers(-2, 10, m)
            offs = np.sort(rng.integers(-3, 400, m)) if rng.random() < 0.7 else rng.integers(-3, 400, m)
            heads = rng.integers(-1, 30, m)
            counts = rng.integers(0, 40, m)
            lay = (ids, offs, heads, counts)
            kept, bad = walk_rule(lay, L)
            got, err = call_walk(emu, lay, L)
            assert got == kept and err == (32 if bad else 0)


# ----------------------------------------------------------------------------------------------------- staging
def stage(emu, lay, clips, cut, N, ws, wl):
    a = [arr(v) for v in lay]
    lengths = arr([c.size for c in clips])
    sig = (ctypes.c_void_p * len(clips))(*[c.ctypes.data for c in clips])
    out = np.full(N + 64, np.nan, np.float32)
    info = np.zeros(3, np.int32)
    b = arr(np.round(np.linspace(0, N, 3)))
    err = emu.emu_bg_stage(b.ctypes.data, N, 3, 2, 2, ws, wl, *[v.ctypes.data for v in a], a[0].size,
                           lengths.ctypes.data, ctypes.cast(sig, vp), int(clips[0].dtype == np.int16), len(clips), cut,
                           out.ctypes.data, info.ctypes.data)
    x0, x1 = int(info[0]), int(info[1])
    return out[:x1 - x0], x0, x1, bool(info[2]), err


@pytest.mark.parametrize("dtype", ["int16", "float32"])
def test_staging_equals_the_assembled_bed(emu, dtype):
    rng = np.random.default_rng(11 if dtype == "int16" else 12)
    clips = []
    for _ in range(6):
        k = int(rng.integers(1, 3000))
        v = rng.uniform(-1, 1, k)
        clips.append((v * 32767).astype(np.int16) if dtype == "int16" else v.astype(np.float32))
    lengths = [c.size for c in clips]
    for t in range(60):
        N = int(rng.integers(3000, 9000))
        cut = N + int(rng.integers(0, 300))
        m = int(rng.integers(1, 12))
        lay = np.full((4, m), -1, np.int64)
        pos = int(rng.integers(0, 500))
        for e in range(m):
            i = int(rng.integers(0, len(clips)))
            h = int(rng.integers(0, lengths[i]))
            c = int(rng.integers(1, lengths[i] - h + 1))
            lay[:, e] = i, pos, h, c
            if rng.random() < 0.1:
                lay[3, e] = 0                           # an invalid one now and then
            pos += c + int(rng.integers(0, 400))
        if t % 7 == 0:
            lay[1, -1] = max(cut, lay[1, -1])              # an entry at or past the cut
        kept, bad = walk_rule(lay, lengths)
        bed = np.zeros(cut, np.float32)
        for i, o, h, c in kept:
            if o < cut:
                n = min(c, cut - o)
                v = clips[i][h:h + n]
                bed[o:o + n] = v.astype(np.float32) / np.float32(32768) if dtype == "int16" else v
        wl = int(rng.integers(100, N // 2))
        ws = int(rng.integers(0, N - wl + 1))
        x, x0, x1, same_view, err = stage(emu, lay, clips, cut, N, ws, wl)
        assert same_view and err == (32 if bad else 0)
        assert np.array_equal(x, bed[x0:x1]) if x1 <= cut else np.array_equal(x[:cut - x0], bed[x0:])


# ------------------------------------------------------------------------------------------------ the generator
def test_layout_rows_are_valid(emu):
    g = torch.Generator().manual_seed(2)
    lengths = torch.randint(1000, 40000, (40,), generator=g)
    for total, m in ((160000, 16), (50000, 3), (8000, 128)):
        ids, offs, heads, counts = dry.background_audio_layouts(lengths, total, m, 400, generator=g)
        assert ids.shape == (400, m) and ids.dtype == torch.int32
        for r in range(400):
            lay = [ids[r].numpy(), offs[r].numpy(), heads[r].numpy(), counts[r].numpy()]
            kept, bad = walk_rule(lay, lengths.tolist())
            assert not bad
            k = len(kept)
            assert (ids[r, :k] >= 0).all() and (ids[r, k:] == -1).all() and (offs[r, k:] == -1).all()
            assert len({i for i, _, _, _ in kept}) == k                       # without replacement
            for e, (i, o, h, c) in enumerate(kept):
                assert o + c <= total
                if h > 0 or c < lengths[i]:
                    assert e == k - 1                                          # only the end clip is trimmed
            assert call_walk(emu, lay, lengths.tolist()) == (kept, 0)


def host_outcome(lens16, json_path, total, sr):
    chosen = dry.get_random_wav_path_from_json(json_path, total, threshold=0.4)
    places, _, _ = dry._place_background_audio([lens16[int(p)] for p in chosen], total, total / sr, sr)
    return outcome([(int(chosen[k]), dst, src, cnt) for k, dst, src, cnt in places], lens16, total)


def outcome(places, lens16, total):
    """(clips placed, the end entry's (clip, lead, trail) or None, its count) of a layout's kept entries."""
    if not places:
        return (0, None)
    last = places[-1]
    trimmed = last[2] > 0 or last[3] < lens16[last[0]]
    return (len(places), (last[0], last[2], last[3]) if trimmed else None)


@pytest.mark.parametrize("different_select", [False, True])
def test_outcome_frequencies_match_the_host_loop(tmp_path, different_select):
    sr = 10                                             # tails of 0..100 samples
    lens16 = [37, 61, 23, 90]
    sel = [(v * 441) // 160 for v in lens16] if different_select else lens16
    js = tmp_path / "bg.json"
    js.write_text(json.dumps({str(i): v for i, v in enumerate(sel)}))
    total = 150
    n = 40000
    random.seed(5)
    host = collections.Counter(host_outcome(lens16, str(js), total, sr) for _ in range(n))
    g = torch.Generator().manual_seed(6)
    ids, offs, heads, counts = dry.background_audio_layouts(torch.tensor(lens16), total, 8, n, generator=g, sample_rate=sr,
                                                            select_lengths=torch.tensor(sel))
    dev = collections.Counter()
    for r in range(n):
        k = int((ids[r] >= 0).sum())
        dev[outcome([(int(ids[r, e]), int(offs[r, e]), int(heads[r, e]), int(counts[r, e])) for e in range(k)],
                    lens16, total)] += 1
    keys = set(host) | set(dev)
    assert len(keys) > 20
    for key in keys:
        p = (host[key] + dev[key]) / (2 * n)
        sd = np.sqrt(2 * p * (1 - p) / n) + 1e-12
        assert abs(host[key] - dev[key]) / n <= 5 * sd + 2.0 / n, (key, host[key], dev[key])
    # and the coarse outcomes by name: clips per bed, an end clip or not
    for f in (lambda k: k[0], lambda k: k[1] is None):
        h, d = collections.Counter(), collections.Counter()
        for key, v in host.items():
            h[f(key)] += v
        for key, v in dev.items():
            d[f(key)] += v
        for key in set(h) | set(d):
            p = (h[key] + d[key]) / (2 * n)
            assert abs(h[key] - d[key]) / n <= 5 * np.sqrt(2 * p * (1 - p) / n) + 2.0 / n, (key, h[key], d[key])


# --------------------------------------------------------------------------------------------- background_clips
def test_background_clips_equal_what_create_background_audio_adds(tmp_path):
    rng = np.random.default_rng(8)
    raw = {"a.wav": (torch.from_numpy(rng.standard_normal((2, 30001)).astype(np.float32) * 0.3), 44100),
           "b.wav": (torch.from_numpy(rng.standard_normal((1, 9000)).astype(np.float32) * 0.3), 16000),
           "c.wav": (torch.from_numpy(rng.standard_normal((2, 7000)).astype(np.float32) * 0.3), 16000)}
    loader = lambda p: (raw[p][0].clone(), raw[p][1])    # noqa: E731
    clips = dry.background_clips(list(raw), 16000, loader)
    assert all(c.dtype == torch.float32 and c.dim() == 1 and not c.is_cuda for c in clips)
    js = tmp_path / "bg.json"
    # one clip per bed: its length reaches 0.4 * total, and a total above it leaves it whole at offset 0 when the tail
    # and trims fall outside it; check the samples it adds over every placement the function made
    for k, p in enumerate(raw):
        js.write_text(json.dumps({p: int(raw[p][0].shape[-1])}))
        for seed in range(6):
            random.seed(seed)
            length = 2.5
            bed, _, _ = dry.create_background_audio(str(js), length, 16000, loader=loader)
            random.seed(seed)
            chosen = dry.get_random_wav_path_from_json(str(js), int(length * 16000), threshold=0.4)
            places, _, _ = dry._place_background_audio([clips[k].numel()], int(length * 16000), length, 16000)
            for _, dst, src, count in places:
                assert torch.equal(bed[0, dst:dst + count], clips[k][src:src + count])
    bad = {"d.wav": (torch.zeros((3, 100)), 16000)}
    with pytest.raises(ValueError, match="shape"):
        dry.background_clips(["d.wav"], 16000, lambda p: bad[p])
