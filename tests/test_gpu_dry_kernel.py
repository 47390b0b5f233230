"""The dry-stream assembly kernel (ss_dry_assemble_dev: k_dry_assemble) called through the C ABI, against the float64
polyphase restatement of torchaudio's Resample in tests/mix_reference.py: every rate pair the dataloaders meet, mono and
stereo, clips from 1 sample to about 10 s placed from every edge of their resampled length, heterogeneous batches and
the argument checks.  Sources, filter banks and the stream sit inside NaN-filled allocations whose guards must stay
NaN, so a read outside the documented read set shows up as NaN and a write outside [0, total) as a lost guard."""
import ctypes

import numpy as np
import pytest
import torch

from mix_reference import F32, RESAMPLE_PAIRS, clip_lengths, max_rel, resample_kernel
from mix_reference import Clip, DryBuf

pytestmark = pytest.mark.gpu

NAN = float("nan")
SS_ERR_INVALID, SS_ERR_UNSUPPORTED = -1, -5
MAX_REL = [0.0]         # largest per-clip max-relative resampling error seen


def res_len(L, orig, new):
    if orig == new:
        return L
    _, o, n, _ = resample_kernel(orig, new)
    return -(-n * L // o)


def assemble(clips, out):
    from sonicsim_b200 import _lib as L
    from sonicsim_b200 import render
    R = render.default_renderer()
    arr = (L.SsDryClip * max(len(clips), 1))(*[c.c for c in clips])
    st = R.lib.ss_dry_assemble_dev(R.ctx, arr, len(clips), ctypes.c_void_p(out.ptr), out.n,
                                   ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return st


def check_stream(clips, out):
    """Every clip's range against its reference, zeros elsewhere, every guard still NaN."""
    y = out.get()
    assert out.guards_nan()
    placed = np.zeros(out.n, bool)
    for c in clips:
        assert c.src.guards_nan()
        got = y[c.dst_start:c.dst_start + c.count]
        placed[c.dst_start:c.dst_start + c.count] = True
        want, bound = c.expected()
        if bound is None:
            assert np.array_equal(got, want), (c.orig, c.ch, c.L, c.src_start, c.count)
            continue
        err = np.abs(got.astype(np.float64) - want)
        assert np.all(err <= bound), (c.orig, c.new, c.ch, c.L, c.src_start, float(np.max(err - bound)))
        if c.count >= 16:         # a single near-zero sample would make the relative figure meaningless
            r = max_rel(got, want)
            MAX_REL[0] = max(MAX_REL[0], r)
            assert r <= 1e-6, (c.orig, c.new, c.ch, c.L, c.src_start, r)
    assert not y[~placed].any() and not np.isnan(y).any()
    return y


def pair_clips(orig, new, ch, rng):
    """Every clip length of clip_lengths, each placed from src_start 0, 1, the middle and res_len - 1 up to exactly its
    end, plus empty clips; placements alternately touching and 3 samples apart, from 0 to exactly `total`."""
    lengths = clip_lengths(orig, new) if orig != new else [1, 2, 3, 5, 160, 10 * orig + 7]
    clips, cursor = [], 0
    for i, L in enumerate(lengths):
        x = (rng.standard_normal((ch, L)) * 0.1).astype(F32)
        n = res_len(L, orig, new)
        for j, s in enumerate(sorted({0, 1, n // 2, n - 1} & set(range(n)))):
            clips.append(Clip(x, orig, new, s, n - s, cursor, off=(i + j) % 4))
            cursor += n - s + (3 if (i + j) % 2 else 0)
        clips.append(Clip(x, orig, new, 0, 0, cursor))
    return clips, cursor


@pytest.mark.parametrize("ch", [1, 2])
@pytest.mark.parametrize("orig,new", [(16000, 16000)] + RESAMPLE_PAIRS)
def test_dry_clips_against_reference(orig, new, ch):
    rng = np.random.default_rng(orig * 3 + new + ch)
    clips, total = pair_clips(orig, new, ch, rng)
    out = DryBuf(total)
    assert assemble(clips, out) == 0
    check_stream(clips, out)


def _batch(rng):
    """About 40 clips of every rate pair and both channel counts, touching, from 0 to exactly `total`."""
    clips, cursor = [], 0
    pairs = [(16000, 16000)] + RESAMPLE_PAIRS
    for i in range(40):
        orig, new = pairs[i % len(pairs)]
        ch = 1 + (i // len(pairs)) % 2
        L = int(rng.choice([1, 2, 37, 441, 1000, 4800]))
        n = res_len(L, orig, new)
        s = int(rng.integers(0, n))
        count = n - s if i % 3 else int(rng.integers(0, n - s + 1))
        clips.append(Clip((rng.standard_normal((ch, L)) * 0.1).astype(F32), orig, new, s, count, cursor, i % 4))
        cursor += count
    return clips, cursor


def test_dry_batch_equals_single_clips():
    clips, total = _batch(np.random.default_rng(40))
    out = DryBuf(total)
    assert assemble(clips, out) == 0
    y = check_stream(clips, out)
    assert clips[0].dst_start == 0 and clips[-1].dst_start + clips[-1].count == total
    for c in clips:
        alone = DryBuf(total, 1)
        assert assemble([c], alone) == 0
        a = alone.get()
        assert alone.guards_nan()
        assert np.array_equal(a[c.dst_start:c.dst_start + c.count], y[c.dst_start:c.dst_start + c.count])
        a[c.dst_start:c.dst_start + c.count] = 0
        assert not a.any()


def test_dry_no_clips_zero_fills_exactly_total():
    out = DryBuf(4097, 3)
    assert assemble([], out) == 0
    assert out.guards_nan() and np.array_equal(out.get(), np.zeros(4097, F32))


def test_dry_refusals_leave_the_stream_untouched():
    rng = np.random.default_rng(8)
    x = (rng.standard_normal((1, 500)) * 0.1).astype(F32)
    n = res_len(500, 44100, 16000)
    ok = [Clip(x, 16000, 16000, 0, 100, 0), Clip(x, 44100, 16000, 0, n, 100)]
    out = DryBuf(1000)
    assert assemble(ok + [Clip(x, 16000, 16000, 0, 50, 100 + n)], out) == 0       # touching ranges are fine
    assert assemble([Clip(x, 44100, 16000, 1, n, 0)], DryBuf(1000)) == SS_ERR_INVALID  # one sample past res_len
    for bad in (Clip(x, 16000, 16000, 0, 50, 99),            # overlaps the first clip's last sample
                Clip(x, 16000, 16000, 0, 10, 150),           # inside the second clip
                Clip(x, 44100, 16000, 0, n, 0)):             # the same range as the first clip and more
        out = DryBuf(1000)
        assert assemble(ok + [bad], out) == SS_ERR_INVALID
        assert np.all(np.isnan(out.t.cpu().numpy()))
    out = DryBuf(1000)
    assert assemble([Clip(x, 16000, 16000, 0, 0, 5)] * 65536, out) == SS_ERR_UNSUPPORTED
    assert np.all(np.isnan(out.t.cpu().numpy()))


def test_report_largest_resampling_error():
    """Runs last in this module: the largest per-clip max-relative error the checks above met."""
    print("largest per-clip max-relative resampling error: %.3g" % MAX_REL[0])
    assert MAX_REL[0] <= 1e-6
