"""Grouped layout draws (ss_layout_group; render.LayoutDraw(groups=, group=); dry.long_audio_layouts(groups=, group=))
on the CPU, through k_layout_grouped's own code (ss_phases.cuh: layout_row_grouped, exported by
tests/emu/ss_emu_layout_group.cu).
  - The defining property, bit for bit: a grouped row over group g equals the ungrouped row of the same (seed, t, r)
    over a pool of group g's utterances alone (k_layout's code, tests/emu/ss_emu_layout.cu) with its ids shifted by
    bounds[g], over many (seed, t, r), 1 to 300 utterances per group and G from 1 to 1000; G = 1 is the ungrouped
    draw; g = -1 and g = G are clamped and flagged; groups where nothing fits give empty rows; a group reaches K = 1024
    exactly.  The emulated rows also equal the Python restatement (tests/layout_reference.py) over the sub-pool.
  - dry.long_audio_layouts(groups=, group=): every id of row i lies in group group[i], and selection counts, first
    gaps and first ids agree with layout_reference's host loops over that group within 5 standard errors.
  - dry.long_audio_max_selected(groups=) is the largest K of the groups; bad bounds are refused.
  - dry.speaker_groups lists, per speaker directory, the files get_random_wav_path walks, in its order.
  - render.LayoutDraw's group refusals are ValueErrors raised before any C call; SsLayoutGroup matches the header.
The kernel itself needs a device: tests/test_gpu_layout_groups.py."""
import ctypes
import os
import random
import re

import numpy as np
import pytest

import group_reference as gr
import layout_reference as lr
from sonicsim_b200 import dry

SEEDS = [(0, 0), (20261018, 7), (-77, 123456789), ((1 << 63) - 1, -1), (-(1 << 63), 1 << 40)]
RATE = 1600


def check_group(lengths, bounds, g, rng_pairs, r, total, m, gap_max=10 * RATE):
    """Grouped rows over group g (clamped when outside [0, G)) equal the sub-pool's plain rows, ids shifted."""
    G = len(bounds) - 1
    c = min(max(g, 0), G - 1)
    lo, hi = int(bounds[c]), int(bounds[c + 1])
    ids, offs, err = gr.grouped_rows(rng_pairs, r, lengths, total, m, gap_max, bounds, g)
    want_ids, want_offs = gr.plain_rows(rng_pairs, r, lengths[lo:hi], total, m, gap_max)
    assert np.array_equal(ids, gr.shifted(want_ids, lo)), (g, r)
    assert np.array_equal(offs, want_offs), (g, r)
    assert err == (0 if 0 <= g < G else 128)
    valid = ids >= 0
    assert ((ids[valid] >= lo) & (ids[valid] < hi)).all()
    return ids, offs


@pytest.mark.parametrize("G,lo,hi", [(1, 1, 300), (2, 1, 300), (7, 1, 300), (100, 1, 40), (1000, 1, 12)])
def test_grouped_rows_are_the_sub_pools_rows(G, lo, hi):
    rng = np.random.default_rng(G)
    sizes = rng.integers(lo, hi + 1, G)
    sizes[rng.integers(0, G)] = hi                         # one group of the most
    sizes[rng.integers(0, G)] = 1                          # one of a single utterance
    lengths, bounds = gr.corpus(G, sizes, int(0.2 * RATE), int(1.5 * RATE))
    pairs = np.array(SEEDS, dtype=np.int64)
    groups = sorted(set([0, G - 1] + rng.integers(0, G, 6).tolist()))
    for total, m in ((12 * RATE, 12), (60 * RATE, 128), (RATE, 1)):
        for r in (0, 1, 37, 4095):
            for g in groups:
                check_group(lengths, bounds, g, pairs, r, total, m)


def test_one_group_is_the_ungrouped_draw():
    lengths, _ = gr.corpus(3, [250], int(0.2 * RATE), int(1.5 * RATE))
    pairs = np.array(SEEDS, dtype=np.int64)
    for r in (0, 5, 300):
        ids, offs, err = gr.grouped_rows(pairs, r, lengths, 30 * RATE, 64, 10 * RATE, [0, 250], 0)
        plain = gr.grouped_rows(pairs, r, lengths, 30 * RATE, 64, 10 * RATE)
        ref = gr.plain_rows(pairs, r, lengths, 30 * RATE, 64, 10 * RATE)
        assert err == 0 and plain[2] == 0
        assert np.array_equal(ids, plain[0]) and np.array_equal(offs, plain[1])
        assert np.array_equal(ids, ref[0]) and np.array_equal(offs, ref[1])


def test_rows_equal_the_python_restatement_of_the_sub_pool():
    lengths, bounds = gr.corpus(11, [5, 40, 1, 17], int(0.2 * RATE), int(1.5 * RATE))
    for (seed, t) in SEEDS:
        for r in (0, 3):
            for g in range(4):
                lo, hi = int(bounds[g]), int(bounds[g + 1])
                ids, offs, _ = gr.grouped_rows([seed, t], r, lengths, 20 * RATE, 16, 10 * RATE, bounds, g)
                (want_ids, want_offs, _, _), _ = lr.layout_row(seed, t, r, lengths[lo:hi].tolist(), 20 * RATE, 16,
                                                               RATE, False)
                assert ids[0].tolist() == [i + lo if i >= 0 else -1 for i in want_ids]
                assert offs[0].tolist() == want_offs


def test_out_of_range_groups_are_clamped_and_flagged():
    lengths, bounds = gr.corpus(5, [30, 8, 20], int(0.2 * RATE), int(1.5 * RATE))
    pairs = np.array(SEEDS, dtype=np.int64)
    for g, c in ((-1, 0), (-(1 << 31), 0), (3, 2), (1 << 30, 2)):
        a = check_group(lengths, bounds, g, pairs, 2, 15 * RATE, 24)
        b = check_group(lengths, bounds, c, pairs, 2, 15 * RATE, 24)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    # one row out of range flags the call, the others are unaffected
    ids, offs, err = gr.grouped_rows(pairs[:3], 2, lengths, 15 * RATE, 24, 10 * RATE, bounds, [1, 3, 0])
    assert err == 128
    for q, g in enumerate([1, 2, 0]):
        one = gr.grouped_rows(pairs[q], 2, lengths, 15 * RATE, 24, 10 * RATE, bounds, g)
        assert np.array_equal(ids[q], one[0][0]) and np.array_equal(offs[q], one[1][0]) and one[2] == 0


def test_groups_where_nothing_fits_give_empty_rows():
    rng = np.random.default_rng(8)
    total = 5 * RATE
    long = rng.integers(total + 1, 3 * total, 9).astype(np.int32)       # no utterance of group 1 fits
    short = rng.integers(RATE // 5, RATE, 12).astype(np.int32)
    lengths = np.concatenate([short, long, short[:3]])
    bounds = [0, 12, 21, 24]
    pairs = np.array(SEEDS, dtype=np.int64)
    ids, offs = check_group(lengths, bounds, 1, pairs, 0, total, 8, gap_max=RATE // 10)
    assert (ids == -1).all() and (offs == -1).all()
    ids, _ = check_group(lengths, bounds, 0, pairs, 0, total, 8, gap_max=RATE // 10)
    assert (ids[:, 0] >= 0).all()                                       # (short gaps: the others' rows are not)


def test_a_group_at_the_cap():
    total = 1024
    lengths = np.concatenate([np.full(40, 300, np.int32), np.ones(1100, np.int32), np.full(9, 5, np.int32)])
    bounds = [0, 40, 1140, 1149]
    assert dry.long_audio_max_selected(lengths, total, bounds) == 1024
    assert dry.long_audio_max_selected(lengths, total + 1, bounds) == 1025
    assert dry.long_audio_max_selected(lengths[:40], total) == 3
    pairs = np.array(SEEDS, dtype=np.int64)
    for m in (1, 128):
        ids, offs = check_group(lengths, bounds, 1, pairs, 9, total, m, gap_max=0)
        assert ((ids >= 0).sum(axis=1) == m).all()                     # 1024 selected, m placed
        check_group(lengths, bounds, 0, pairs, 9, total, m, gap_max=0)
        check_group(lengths, bounds, 2, pairs, 9, total, m, gap_max=0)


def test_max_selected_over_groups_and_bad_bounds():
    lengths, bounds = gr.corpus(2, [10, 3, 50], 100, 900)
    want = max(dry.long_audio_max_selected(lengths[lo:hi], 2000) for lo, hi in zip(bounds[:-1], bounds[1:]))
    assert dry.long_audio_max_selected(lengths, 2000, bounds) == want
    assert dry.long_audio_max_selected(lengths, 2000, [0, lengths.size]) == dry.long_audio_max_selected(lengths, 2000)
    import torch
    assert dry.long_audio_max_selected(torch.from_numpy(lengths), 2000, torch.from_numpy(bounds)) == want
    for bad in ([1, 63], [0, 62], [0, 10, 10, 63], [0, 20, 10, 63], [0], [[0, 63]], [0.0, 63.5]):
        with pytest.raises(ValueError):
            dry.long_audio_max_selected(lengths, 2000, bad)


# ------------------------------------------------------------------------------------- torch form in distribution
def test_torch_layouts_follow_the_rule_over_each_group():
    import torch
    total, sr, m = 6 * RATE, RATE, 12
    lengths, bounds = gr.corpus(21, [6, 1, 9, 4], int(0.5 * RATE), int(2.5 * RATE))
    count = 24000
    group = torch.arange(count) % 4
    g = torch.Generator().manual_seed(5)
    K = dry.long_audio_max_selected(lengths, total, bounds)
    for max_selected in (None, K):
        ids, offs = dry.long_audio_layouts(torch.from_numpy(lengths), total, m, count, generator=g, sample_rate=sr,
                                           max_selected=max_selected, groups=bounds, group=group)
        ids, offs = ids.numpy(), offs.numpy()
        random.seed(17)
        for q in range(4):
            lo, hi = int(bounds[q]), int(bounds[q + 1])
            rows = ids[q::4]
            valid = rows >= 0
            assert ((rows[valid] >= lo) & (rows[valid] < hi)).all()      # every id in its group
            host = [lr.host_stream(lengths[lo:hi].tolist(), total, sr) for _ in range(count // 4)]
            a_n, b_n = valid.sum(axis=1), np.array([len(h) for h in host])
            a_gap = offs[q::4][valid[:, 0], 0]
            b_gap = np.array([h[0][1] for h in host if h])
            a_id = rows[valid[:, 0], 0] - lo
            b_id = np.array([h[0][0] for h in host if h])
            for a, b in ((a_n, b_n), (a_gap, b_gap)):
                se = np.sqrt(a.var() / a.size + b.var() / b.size) + 1e-12
                assert abs(a.mean() - b.mean()) < 5 * se, (q, a.mean(), b.mean())
            for i in range(hi - lo):
                pa, pb = (a_id == i).mean(), (b_id == i).mean()
                se = np.sqrt(pa * (1 - pa) / a_id.size + pb * (1 - pb) / b_id.size) + 1e-12
                assert abs(pa - pb) < 5 * se, (q, i, pa, pb)


def test_torch_layouts_clamp_groups_and_keep_the_ungrouped_bits():
    import torch
    lengths, bounds = gr.corpus(4, [5, 7], 100, 400)
    L = torch.from_numpy(lengths)
    ids, _ = dry.long_audio_layouts(L, 2000, 8, 64, generator=torch.Generator().manual_seed(1), groups=bounds,
                                    group=torch.tensor([-5, 9] * 32))
    ids = ids.numpy()
    assert ((ids[0::2] < 5) & (ids[0::2] >= -1)).all() and ((ids[1::2] >= 5) | (ids[1::2] == -1)).all()
    # without groups the call draws what it drew before: the same generator state, the same bits
    a = dry.long_audio_layouts(L, 2000, 8, 64, generator=torch.Generator().manual_seed(2))
    b = dry.long_audio_layouts(L, 2000, 8, 64, generator=torch.Generator().manual_seed(2))
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    for kw in (dict(groups=bounds), dict(group=torch.zeros(64, dtype=torch.int64)),
               dict(groups=bounds, group=torch.zeros(63, dtype=torch.int64)),
               dict(groups=bounds, group=torch.zeros(64)), dict(groups=[0, 5, 11], group=torch.zeros(64).long())):
        with pytest.raises(ValueError):
            dry.long_audio_layouts(L, 2000, 8, 64, **kw)


# ------------------------------------------------------------------------------------------------ speaker groups
def test_speaker_groups_list_the_files_get_random_wav_path_walks(tmp_path, monkeypatch):
    from oracle import dry_fixture
    monkeypatch.setattr(os, "walk", dry_fixture.sorted_walk(os.walk))
    dirs, loaders = [], []
    for name in ("a", "b", "c"):
        (tmp_path / name).mkdir()
        spk, _, loader = dry_fixture.build(tmp_path / name)
        dirs.append(spk)
        loaders.append(loader)
    (tmp_path / "a" / "spk" / "chapter2").mkdir()                      # a second chapter of speaker a
    (tmp_path / "a" / "spk" / "chapter2" / "61-0000.flac").write_bytes(b"")
    paths, bounds = dry.speaker_groups(dirs)
    assert bounds == [0, 15, 29, 43] and len(paths) == 43
    for g, (spk, loader) in enumerate(zip(dirs, loaders)):
        group = paths[bounds[g]:bounds[g + 1]]
        assert all(p.startswith(spk + os.sep) and not p.endswith(".txt") for p in group)
        seen = []
        real_choice = random.choice

        def choice(seq):
            if not seen:
                seen.append(list(seq))
            return real_choice(seq)
        monkeypatch.setattr(random, "choice", choice)
        random.seed(g)
        chosen = dry.get_random_wav_path(spk, 10 ** 9, loader=loader)
        monkeypatch.setattr(random, "choice", real_choice)
        assert seen[0] == group                                      # the same files, in its order
        assert sorted(chosen) == sorted(group)
    empty = tmp_path / "empty"
    (empty / "chapter").mkdir(parents=True)
    (empty / "chapter" / "x.trans.txt").write_text("x")
    with pytest.raises(ValueError):
        dry.speaker_groups(dirs + [str(empty)])
    with pytest.raises(ValueError):
        dry.speaker_groups([])


# ---------------------------------------------------------------------------------------------------- refusals
class _Pool:
    def __init__(self, sizes):
        self.sizes, self.n = list(sizes), len(sizes)


def test_layout_group_refusals_before_any_c_call():
    import torch
    from sonicsim_b200 import render
    R = object.__new__(render.Renderer)                    # no context: a refusal must come before any C call
    R.device, R.lib = 0, None
    cpu = torch.zeros(4, dtype=torch.int32)
    utts, clips = _Pool([100] * 6), _Pool([100] * 4)
    srcs = [render.Pooled(None, cpu[:1], (0, 10), 0, render.DryStream(utts, cpu, cpu)),
            render.Pooled(None, cpu[:1], (0, 10), 0, render.BackgroundStream(clips, cpu, cpu, cpu, cpu))]
    rng = torch.zeros(2, dtype=torch.int64)

    def refused(d, match):
        with pytest.raises(ValueError, match=match):
            R._device_layouts([d], srcs, (None,) * 4, [], [])

    refused(render.LayoutDraw(1, rng, 1000, groups=[0, 4], group=cpu[:1]), "bed slot")
    refused(render.LayoutDraw(0, rng, 1000, groups=[0, 6]), "both")
    refused(render.LayoutDraw(0, rng, 1000, group=cpu[:1]), "both")
    for bad in ([0, 5], [1, 6], [0, 3, 3, 6], [0, 4, 2, 6], [6], np.zeros((2, 2), np.int64)):
        refused(render.LayoutDraw(0, rng, 1000, groups=bad, group=cpu[:1]), "groups must")
    refused(render.LayoutDraw(0, rng, 1000, groups=[0, 2, 6], group=cpu[:1]), "CUDA")
    # positional construction of the fields before groups still works
    d = render.LayoutDraw(0, rng, 1000, 16000, None)
    assert d.groups is None and d.group is None


def test_ss_layout_group_matches_the_header():
    from sonicsim_b200 import _lib
    head = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include",
                             "sonicsim_b200.h")).read()
    body = re.search(r"typedef struct \{([^}]*)\} ss_layout_group;", head).group(1)
    fields = re.findall(r"^\s*(?:const )?(\w+)(\*?)\s+(\w+);", body, re.M)
    assert [f[2] for f in fields] == [n for n, _ in _lib.SsLayoutGroup._fields_]
    want = {"int32_t": ctypes.c_int32}
    for (ty, ptr, name), (_, cty) in zip(fields, _lib.SsLayoutGroup._fields_):
        assert cty is (ctypes.c_void_p if ptr else want[ty]), name
    assert ctypes.sizeof(_lib.SsLayoutGroup) == 24
    assert [getattr(_lib.SsLayoutGroup, n).offset for n, _ in _lib.SsLayoutGroup._fields_] == [0, 4, 8, 16]
