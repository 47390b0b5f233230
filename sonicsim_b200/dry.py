"""Dry-stream assembly (SURVEY 8f rank 2): drop-ins for SonicSim_audio.get_random_wav_path (:152-190),
get_random_wav_path_from_json (:192-228), create_long_audio (:231-279) and create_background_audio (:281-340).

File selection and placement are host logic drawn from the `random` module in exactly the reference's order, so a
seeded run selects and places the same files.  The arithmetic - resampling, stereo -> mono, adding the clips into
the stream - runs on the CPU through torch like the reference by default, or, with `device=`, in one CUDA kernel
(ss_dry_assemble_dev, csrc/ss_dry.cu) that leaves the stream in HBM for the renderer's device path.

`loader(path) -> (Tensor (channels, n), sample_rate)` defaults to torchaudio.load.
"""
import json
import os
import random
import typing as T


def _default_loader(path):
    import torchaudio
    return torchaudio.load(path)


def _load_resampled(path, sample_rate, loader):
    import torchaudio
    waveform, sr = loader(path)
    if sr != sample_rate:
        waveform = torchaudio.transforms.Resample(orig_freq=sr, new_freq=sample_rate)(waveform)
    return waveform


def _wav_candidates(audio_dir: str) -> T.List[str]:
    """The files get_random_wav_path draws from: every file of the tree but the .txt ones, in os.walk order."""
    return [os.path.join(root, name) for root, _, names in os.walk(str(audio_dir)) for name in names
            if not name.endswith(".txt")]


def get_random_wav_path(audio_dir: str, length: int, threshold: float = 0.9, loader=None) -> T.List[str]:
    """:152-190 - random files of a directory tree whose total length lands in [threshold*length, length]."""
    loader = loader or _default_loader
    candidates = _wav_candidates(audio_dir)
    print(f"audio_path_list: {len(candidates)}")
    n_samples = {p: loader(p)[0].shape[-1] for p in candidates}
    chosen, total = [], 0
    while candidates and total < length * threshold:
        pick = random.choice(candidates)
        if total + n_samples[pick] > length:
            break
        chosen.append(pick)
        total += n_samples[pick]
        candidates.remove(pick)
    return chosen


def get_random_wav_path_from_json(json_dir: str, length: int, threshold: float = 0.9) -> T.List[str]:
    """:192-228 - same from a {path: n_samples} JSON; the file that overshoots is still taken, then it stops."""
    with open(json_dir) as f:
        n_samples = json.load(f)
    candidates = list(n_samples.keys())
    chosen, total = [], 0
    while candidates and total < length * threshold:
        pick = random.choice(candidates)
        chosen.append(pick)
        if not (total + n_samples[pick] < length):
            break
        total += n_samples[pick]
        candidates.remove(pick)
    return chosen


def _resampled_len(n: int, sr: int, sample_rate: int) -> int:
    """Length of torchaudio.transforms.Resample(sr, sample_rate)(x) for x of n samples: ceil(new * n / orig)."""
    if sr == sample_rate:
        return n
    import math
    g = math.gcd(int(sr), int(sample_rate))
    o, nw = int(sr) // g, int(sample_rate) // g
    return -((-nw * n) // o)


def _place_long_audio(lens: T.List[int], total: int, sample_rate: int):
    """The placement loop of create_long_audio (:258-277) on clip lengths alone; same `random` draws.
    Returns (placements [(clip, dst_start, src_start, count)], spans, order of clips used)."""
    alive = list(range(len(lens)))
    places, spans, used, cursor = [], [], [], 0
    while cursor < total and alive:
        k = random.randint(0, len(alive) - 1)
        gap = random.randint(0, int(10 * sample_rate))
        n = gap + lens[alive[k]]
        if cursor + n > total:
            break
        spans.append((cursor + gap, cursor + n))
        places.append((alive[k], cursor + gap, 0, lens[alive[k]]))
        cursor += n
        used.append(alive.pop(k))
    return places, spans, used


def _place_background_audio(lens: T.List[int], total: int, length: float, sample_rate: int):
    """The placement loop of create_background_audio (:305-338) on clip lengths alone; same `random` draws."""
    alive = list(range(len(lens)))
    places, spans, used, cursor = [], [], [], 0
    while cursor < total and alive:
        k = random.randint(0, len(alive) - 1)
        ln = lens[alive[k]]
        tail = random.randint(0, int(10 * sample_rate))
        n = ln + tail
        if n >= total - cursor:                                   # this clip reaches the end of the bed
            slack = int((length * sample_rate - cursor) * 0.1)
            lead, trail = random.randint(0, slack), random.randint(0, slack)
            spans.append((lead + cursor, total - trail))
            # long_audio[:, lead+cursor : total-trail] += padded[:, lead : total-trail-cursor]; beyond the clip the
            # padding is zeros (the slices always have equal length here, so the reference's bare except never fires)
            count = min(ln, total - trail - cursor) - lead
            if count > 0:
                places.append((alive[k], lead + cursor, lead, count))
            used.append(alive.pop(k))
            break
        spans.append((cursor, cursor + n))
        places.append((alive[k], cursor, 0, ln))
        cursor += n
        used.append(alive.pop(k))
    return places, spans, used


def speaker_groups(speaker_dirs) -> T.Tuple[T.List[str], T.List[int]]:
    """An utterance corpus in speaker order, for grouped stream layouts (long_audio_layouts(groups=), render.LayoutDraw
    (groups=)): (paths, bounds).  For each directory of `speaker_dirs` (e.g. the lines of SonicSet's
    {mode}_speech.txt, one LibriSpeech speaker each), the files get_random_wav_path would draw from, in its order
    (os.walk, .txt files left out); paths concatenates them and bounds (G + 1 ints, 0 = bounds[0] < ... < bounds[G] =
    len(paths)) delimits speaker g's files as paths[bounds[g]:bounds[g + 1]].  A pool built from paths in this order
    (one signal per path) has these bounds as its groups.  A directory without such files raises ValueError."""
    paths, bounds = [], [0]
    for d in speaker_dirs:
        files = _wav_candidates(d)
        if not files:
            raise ValueError("speaker_groups: %s holds no file get_random_wav_path would draw" % (d,))
        paths += files
        bounds.append(len(paths))
    if len(bounds) < 2:
        raise ValueError("speaker_groups: need at least one speaker directory")
    return paths, bounds


def _group_bounds(groups, n: int, api: str):
    """`groups` (G + 1 bounds: a host sequence, array or tensor) as an int64 NumPy array, checked to ascend strictly
    from 0 to n."""
    import numpy as np
    b = np.asarray(groups.cpu() if hasattr(groups, "cpu") else groups)
    if b.ndim != 1 or b.size < 2 or not (np.issubdtype(b.dtype, np.integer) or b.dtype == object):
        raise ValueError("%s: groups must be G + 1 >= 2 integer bounds, got %r" % (api, groups))
    b = b.astype(np.int64)
    if b[0] != 0 or b[-1] != n or (np.diff(b) < 1).any():
        raise ValueError("%s: groups must ascend strictly from 0 to the %d utterances of the pool" % (api, n))
    return b


def long_audio_max_selected(lengths, total: int, groups=None) -> int:
    """The most utterances of `lengths` that get_random_wav_path's selection can take for a stream of `total` samples:
    the largest k whose k shortest utterances fit in `total` (at least 1).  With `groups` (G + 1 bounds, see
    speaker_groups), the largest such k over the groups, each of which a row selects from alone.  A host computation,
    once per corpus, for long_audio_layouts(..., max_selected=)."""
    import numpy as np
    v = np.asarray(lengths.cpu() if hasattr(lengths, "cpu") else lengths, dtype=np.int64).reshape(-1)
    b = [0, v.size] if groups is None else _group_bounds(groups, v.size, "long_audio_max_selected")
    return max(max(1, int(np.searchsorted(np.cumsum(np.sort(v[lo:hi])), int(total), side="right")))
               for lo, hi in zip(b[:-1], b[1:]))


def background_audio_max_selected(select_lengths, total: int) -> int:
    """The most clips that get_random_wav_path_from_json's selection (threshold 0.4) can take for a bed of `total`
    samples over clips of `select_lengths`: the most whose running total stays below 0.4 * total, plus the one that
    crosses it (at most n).  A host computation, once per corpus; render.LayoutDraw refuses beds above 1024."""
    import numpy as np
    v = np.sort(np.asarray(select_lengths.cpu() if hasattr(select_lengths, "cpu") else select_lengths,
                           dtype=np.int64).reshape(-1))
    below = int(np.count_nonzero(np.cumsum(v).astype(np.float64) < 0.4 * int(total)))
    return min(v.size, below + 1)


def _long_audio_selection(lengths, total: int, count: int, width: int, kw, lo=None, hi=None):
    """get_random_wav_path's selection, `count` times: (sel, chosen), both (count, width).  sel[r] is the first width
    utterances of a uniform random order, chosen[r] marks its selected prefix (taken while the running total is below
    0.9 * total, up to the first that would overflow `total`).  With lo and hi ((count,) tensors), row r selects from
    utterances [lo[r], hi[r]) only: the others sort behind them and are never chosen."""
    import torch
    keys = torch.rand((count, lengths.numel()), **kw)
    if lo is not None:
        idx = torch.arange(lengths.numel(), device=keys.device)
        keys.masked_fill_((idx < lo[:, None]) | (idx >= hi[:, None]), 2.0)
    if width < lengths.numel():                       # the first `width` of the random order
        sel = torch.topk(keys, width, dim=1, largest=False, sorted=True).indices
    else:
        sel = torch.argsort(keys, dim=1)
    del keys
    ls = lengths[sel]
    cs = torch.cumsum(ls, dim=1)
    take = ((cs - ls).double() < 0.9 * total) & (cs <= total)
    if lo is not None:
        take &= (sel >= lo[:, None]) & (sel < hi[:, None])
    return sel, torch.cumprod(take.to(torch.int8), dim=1).bool()


def long_audio_layouts(lengths, total: int, m: int, count: int, generator=None, sample_rate: int = 16000,
                       max_selected: T.Optional[int] = None, groups=None, group=None):
    """`count` layouts of create_long_audio streams (:231-277) over utterances of `lengths` (a 1-D integer tensor of n
    lengths in samples, already at `sample_rate`), for render.DryStream: (ids, offsets), two int32 tensors of shape
    (count, m) on `lengths`' device.  Torch ops only, so a training step refreshes them on the GPU without a host
    synchronisation; `generator` (of that device) makes them reproducible.

    Each row draws the arrangement create_long_audio would build for a stream of `total` samples:
      - selection, get_random_wav_path's rule: utterances in a uniform random order without replacement, taken while
        the running total is below 0.9 * total, stopping at the first one that would overflow `total`;
      - placement, _place_long_audio's rule: the selected utterances in an independent uniform random order, each
        preceded by a gap uniform in {0, ..., 10 * sample_rate}, placed while the stream's cursor stays within `total`.
    The placement order is drawn afresh rather than reusing the selection order: given the selected set, the selection
    order is not uniform (the stop rule reads its prefix sums), and the reference's placement order is.  The layouts
    match the reference in distribution, not in its `random`-stream draws.  Unused entries are -1 (empty).  A row that
    would place more than m utterances keeps its first m (in stream order), so choose m above total / (shortest
    utterance + 10 * sample_rate / 2) with some margin when that matters.

    Cost: the selection draws one float32 key per (row, utterance).  Without `max_selected` it sorts all n keys of
    every row, and its temporaries peak at about 42 bytes per (row, utterance): 1.5 GB and 7.6 ms on an H100 for
    count = 128 rows over a LibriSpeech-sized n = 2.8e5 (DESIGN section 6).  `max_selected`
    (long_audio_max_selected(lengths, total), computed once per corpus) bounds how many utterances a row can select;
    the call then keeps only the max_selected smallest keys of each row (torch.topk) and works on (count,
    max_selected) and (count, m) tensors behind the (count, n) keys, with the same distribution: 145 MB (the keys)
    and 1.1 ms there.  A bound below long_audio_max_selected's cuts rows short and changes the distribution.

    Speaker groups, as SonicSet builds every stream from one speaker's utterances: `groups` (G + 1 host bounds, 0 =
    groups[0] < ... < groups[G] = n, see speaker_groups) splits the utterances into G contiguous groups, and `group`
    (a (count,) integer tensor on `lengths`' device, e.g. a ValueDraw of distinct speakers) names row i's group.  Row
    i then follows the rule above over the utterances [groups[g], groups[g + 1]) of g = group[i] alone, its ids
    numbered in the whole pool; a group outside [0, G) is clamped into range, as a plan's grouped LayoutDraw clamps
    it.  This matches the plan's grouped draws in distribution.  `max_selected` stays a bound over every group
    (long_audio_max_selected(lengths, total, groups)).  Without groups every row selects from all n utterances, which
    over a multi-speaker corpus strings together utterances of about as many speakers as the stream holds."""
    import torch
    lengths = lengths.reshape(-1).to(torch.int64)
    n, dev = lengths.numel(), lengths.device
    if n < 1 or not 1 <= m <= 128 or count < 1 or (max_selected is not None and max_selected < 1):
        raise ValueError("long_audio_layouts: need n >= 1 utterances, 1 <= m <= 128, count >= 1 and max_selected "
                         ">= 1, got n = %d, m = %d, count = %d, max_selected = %r" % (n, m, count, max_selected))
    lo = hi = None
    if (groups is None) != (group is None):
        raise ValueError("long_audio_layouts: give both groups and group, or neither")
    if groups is not None:
        b = _group_bounds(groups, n, "long_audio_layouts")
        if not isinstance(group, torch.Tensor) or group.numel() != count or group.device != dev or \
                group.dtype.is_floating_point or group.dtype.is_complex or group.dtype == torch.bool:
            raise ValueError("long_audio_layouts: group must be a (count,) integer tensor on the device of lengths")
        bt = torch.from_numpy(b).to(dev)
        g = group.reshape(-1).to(torch.int64).clamp(0, b.size - 2)
        lo, hi = bt[g], bt[g + 1]
    kw = {"generator": generator, "device": dev}
    width = n if max_selected is None else min(n, int(max_selected))
    sel, chosen = _long_audio_selection(lengths, total, count, width, kw, lo, hi)
    # placement: the first m of the chosen ones in a fresh random order, each behind a gap, while the cursor stays
    # within `total` (a row keeps at most m, and what it keeps is a prefix of that order)
    w = min(width, m)
    key = torch.rand((count, width), **kw).masked_fill(~chosen, 2.0)
    order = torch.topk(key, w, dim=1, largest=False, sorted=True).indices
    ids = sel.gather(1, order)
    valid = chosen.gather(1, order)
    lp = lengths[ids]
    gaps = torch.randint(0, int(10 * sample_rate) + 1, (count, w), **kw)
    cur = torch.cumsum((gaps + lp) * valid, dim=1)
    placed = torch.cumprod((valid & (cur <= total)).to(torch.int8), dim=1).bool()
    offsets = cur - lp
    out_ids = torch.full((count, m), -1, dtype=torch.int32, device=dev)
    out_off = torch.full((count, m), -1, dtype=torch.int32, device=dev)
    out_ids[:, :w] = torch.where(placed, ids, -1).to(torch.int32)
    out_off[:, :w] = torch.where(placed, offsets, -1).to(torch.int32)
    return out_ids, out_off


def background_audio_layouts(lengths, total: int, m: int, count: int, generator=None, sample_rate: int = 16000,
                             select_lengths=None):
    """`count` layouts of create_background_audio beds (:281-340) over clips of `lengths` (a 1-D integer tensor of n
    lengths in samples, already at `sample_rate`), for render.BackgroundStream: (ids, offsets, heads, counts), four
    int32 tensors of shape (count, m) on `lengths`' device, -1 in unused entries.  Torch ops only, so a training step
    refreshes them on the GPU without a host synchronisation; `generator` (of that device) makes them reproducible.

    Each row draws the bed create_background_audio would build for `total` samples:
      - selection, get_random_wav_path_from_json's rule with threshold 0.4: clips in a uniform random order without
        replacement, taken while the running total of `select_lengths` (default `lengths`) is below 0.4 * total; the
        clip whose addition reaches `total` is still taken, and selection stops there.  SonicSet's JSONs list clips at
        their native rate (44.1 kHz) and the reference compares those against the 16 kHz total: pass them as
        `select_lengths` to keep that;
      - placement, _place_background_audio's rule: the selected clips in an independent uniform random order, each
        followed by a tail uniform in {0, ..., 10 * sample_rate}.  The first clip whose length plus tail reaches the
        remaining samples is the end clip: with slack = floor((total - cursor) * 0.1), lead and trail uniform in
        {0, ..., slack}, its samples [lead, lead + count) go to cursor + lead, count = min(len, total - trail - cursor)
        - lead, if count > 0, and the row ends there.
    The layouts match the reference in distribution, not in its `random`-stream draws.  A row that would need more than
    m entries keeps its first m (in stream order); beds hold a few clips of tens of seconds, so a small m suffices.

    Cost: one float32 key per (row, clip) for the selection and one for the placement order; background corpora hold
    thousands of clips, so every key of every row is sorted."""
    import torch
    lengths = lengths.reshape(-1).to(torch.int64)
    sl = lengths if select_lengths is None else select_lengths.reshape(-1).to(device=lengths.device, dtype=torch.int64)
    n, dev = lengths.numel(), lengths.device
    if n < 1 or sl.numel() != n or not 1 <= m <= 128 or count < 1:
        raise ValueError("background_audio_layouts: need n >= 1 clips with as many select_lengths, 1 <= m <= 128 and "
                         "count >= 1, got n = %d, %d select_lengths, m = %d, count = %d" % (n, sl.numel(), m, count))
    kw = {"generator": generator, "device": dev}
    sel = torch.argsort(torch.rand((count, n), **kw), dim=1)
    ls = sl[sel]
    # clip i of the order is taken while the total before it is below 0.4 * total (a prefix: the totals only grow, and
    # the one that reaches `total` ends the selection with every later total above 0.4 * total)
    chosen = (torch.cumsum(ls, dim=1) - ls).double() < 0.4 * total
    w = min(n, m)
    key = torch.rand((count, n), **kw).masked_fill(~chosen, 2.0)
    order = torch.topk(key, w, dim=1, largest=False, sorted=True).indices
    ids = sel.gather(1, order)
    valid = chosen.gather(1, order)
    lp = lengths[ids]
    tails = torch.randint(0, int(10 * sample_rate) + 1, (count, w), **kw)
    span = (lp + tails) * valid
    cum = torch.cumsum(span, dim=1)
    cursor = cum - span
    reach = valid & (cum >= total)                       # the end clip is the first valid one that reaches `total`
    end = reach & (torch.cumsum(reach.to(torch.int32), dim=1) == 1)
    whole = valid & ~reach                               # (every valid clip before the end clip)
    slack = torch.floor((total - cursor).double() * 0.1)
    lead = torch.minimum(torch.floor(torch.rand((count, w), dtype=torch.float64, **kw) * (slack + 1)), slack).long()
    trail = torch.minimum(torch.floor(torch.rand((count, w), dtype=torch.float64, **kw) * (slack + 1)), slack).long()
    cnt_end = torch.minimum(lp, total - trail - cursor) - lead
    keep_end = end & (cnt_end > 0)
    keep = (whole & (lp > 0)) | keep_end
    out = [torch.full((count, m), -1, dtype=torch.int32, device=dev) for _ in range(4)]
    out[0][:, :w] = torch.where(keep, ids, -1).to(torch.int32)
    out[1][:, :w] = torch.where(keep, torch.where(keep_end, cursor + lead, cursor), -1).to(torch.int32)
    out[2][:, :w] = torch.where(keep, torch.where(keep_end, lead, 0), -1).to(torch.int32)
    out[3][:, :w] = torch.where(keep, torch.where(keep_end, cnt_end, lp), -1).to(torch.int32)
    return tuple(out)


def background_clips(paths, sample_rate: int = 16000, loader=None):
    """The clips of a background corpus as 1-D float32 CPU tensors, each exactly the signal create_background_audio
    adds for its path: resampled to `sample_rate` (_load_resampled) and, when stereo, averaged to mono.  A clip of any
    other channel count than 1 or 2 raises ValueError.  A float32 or 16-bit dry pool of render.BackgroundStream beds is
    built from these."""
    import torch
    loader = loader or _default_loader
    out = []
    for p in paths:
        clip = _load_resampled(p, sample_rate, loader)
        if clip.dim() != 2 or clip.shape[0] not in (1, 2):
            raise ValueError("background_clips: %s has shape %s, need (1, n) or (2, n)" % (p, tuple(clip.shape)))
        if clip.shape[0] == 2:
            clip = clip.mean(dim=0, keepdim=True)
        out.append(clip[0].to(torch.float32).contiguous())
    return out


_kernel_cache: T.Dict[T.Tuple[int, int, str], T.Tuple] = {}


def _resample_kernel(sr: int, sample_rate: int, device):
    """torchaudio's own polyphase filter bank for Resample(sr, sample_rate), transposed to (taps, new) on `device`."""
    key = (int(sr), int(sample_rate), str(device))
    if key not in _kernel_cache:
        import math
        import torchaudio
        rs = torchaudio.transforms.Resample(orig_freq=sr, new_freq=sample_rate)
        g = math.gcd(int(sr), int(sample_rate))
        kt = rs.kernel[:, 0, :].t().contiguous().to(device)       # (taps, new)
        _kernel_cache[key] = (kt, int(sr) // g, int(sample_rate) // g, int(rs.width))
    return _kernel_cache[key]


def _assemble_device(raw, places, total: int, sample_rate: int, device):
    """Resample + stereo mean + placement of the drawn clips in one kernel (ss_dry_assemble_dev); returns a
    (1, total) float32 tensor on `device`."""
    import ctypes
    import torch
    from . import _lib
    from .render import Renderer, default_renderer
    dev = torch.device(device)
    if dev.type != "cuda":
        raise ValueError("dry-stream assembly on a device needs a CUDA device, got %r" % (device,))
    index = dev.index if dev.index is not None else torch.cuda.current_device()
    dev = torch.device("cuda", index)
    R = default_renderer()
    if R.device != index:                                         # a context of the library on the stream's own GPU
        R = Renderer(index)
    out = torch.empty((1, total), dtype=torch.float32, device=dev)
    n = len(places)
    clips = (_lib.SsDryClip * max(n, 1))()
    keep = []
    for i, (k, dst, src, count) in enumerate(places):
        wav, sr = raw[k]
        w = wav.to(dtype=torch.float32).contiguous()
        w = (w.pin_memory() if not w.is_cuda else w).to(dev, non_blocking=True)
        keep.append(w)
        kt, o, nw, width, taps = None, 1, 1, 0, 1
        if sr != sample_rate:
            kt, o, nw, width = _resample_kernel(sr, sample_rate, dev)
            taps = 2 * width + o
        clips[i] = _lib.SsDryClip(src=w.data_ptr(), kernel_t=kt.data_ptr() if kt is not None else None, dst_start=dst,
                                  src_start=src, count=count, channels=w.shape[0], src_len=w.shape[-1], orig=o,
                                  new_rate=nw, width=width, taps=taps)
    _lib.check(R.lib.ss_dry_assemble_dev(R.ctx, clips, n, ctypes.c_void_p(out.data_ptr()), total,
                                         ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    for w in keep:                                               # the kernel reads the clips asynchronously
        w.record_stream(torch.cuda.current_stream(dev))
    return out


def create_long_audio(audio_path: str, length: float, sample_rate: int = 16000, loader=None, device=None):
    """:231-279 - utterances of one speaker laid end to end, each preceded by 0-10 s of silence.
    Returns (long_audio (1, length*sr), [(start, end), ...], [path, ...]).  With `device` (a CUDA device) the clips
    are resampled and placed by the GPU and the stream is returned as a device tensor; selection and placement
    consume the `random` stream exactly as without it."""
    import torch
    loader = loader or _default_loader
    print("create_long_audio: ", audio_path)
    total = int(length * sample_rate)
    paths = get_random_wav_path(audio_path, total, loader=loader)
    if device is not None:
        raw = [loader(p) for p in paths]
        lens = [_resampled_len(w.shape[-1], sr, sample_rate) for w, sr in raw]
        places, spans, used = _place_long_audio(lens, total, sample_rate)
        return _assemble_device(raw, places, total, sample_rate, device), spans, [paths[k] for k in used]
    clips = [_load_resampled(p, sample_rate, loader) for p in paths]
    long_audio = torch.zeros((1, total), device=clips[0].device)
    places, spans, used = _place_long_audio([c.shape[-1] for c in clips], total, sample_rate)
    for k, dst, src, count in places:
        long_audio[:, dst:dst + count] += clips[k][:, src:src + count]
    return long_audio, spans, [paths[k] for k in used]


def create_background_audio(audio_path: str, length: float, sample_rate: int = 16000, loader=None, device=None):
    """:281-340 - noise / music bed from a {path: n_samples} JSON: clips (stereo averaged to mono) followed by
    0-10 s of silence; the clip that reaches the end is trimmed by up to 10 % of the remainder on both sides.
    `device`: as for create_long_audio."""
    import torch
    loader = loader or _default_loader
    print("create_background_audio: ", audio_path)
    total = int(length * sample_rate)
    paths = get_random_wav_path_from_json(audio_path, total, threshold=0.4)
    if device is not None:
        raw = [loader(p) for p in paths]
        lens = [_resampled_len(w.shape[-1], sr, sample_rate) for w, sr in raw]
        places, spans, used = _place_background_audio(lens, total, length, sample_rate)
        return _assemble_device(raw, places, total, sample_rate, device), spans, [paths[k] for k in used]
    clips = [_load_resampled(p, sample_rate, loader) for p in paths]
    long_audio = torch.zeros((1, total), device=clips[0].device)
    places, spans, used = _place_background_audio([c.shape[-1] for c in clips], total, length, sample_rate)
    for k, dst, src, count in places:
        clip = clips[k]
        if clip.shape[0] == 2:
            clip = clip.mean(dim=0, keepdim=True)
        long_audio[:, dst:dst + count] += clip[:, src:src + count]
    return long_audio, spans, [paths[k] for k in used]
