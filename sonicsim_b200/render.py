"""Batch-level entry points (additive - NOT reference API, see SURVEY section 0 / D1).

`convolve_moving` and `render_scene` are the names BASELINE.json's north star uses; the reference
has no such symbols.  They render many (utterance, source) units with one C-ABI call
(ss_render_host / ss_render_dev) instead of the reference's serial per-source loop
(SonicSet.py:77-94).  Host arrays in / out by default; `Renderer.render_device` takes CUDA tensors.
"""
import collections
import ctypes
import math
import typing as T
import weakref

import numpy as np

from . import _lib
from ._lib import SsPostLufs, SsSource
from .SonicSim_moving import _as_f32, _samples_per_interval, bounds_from_counts


class MovingSource(T.NamedTuple):
    """One moving source: dry (N,), RIRs (P, C, L), trajectory as int32 segment bounds (P,).
    `bounds_host` (device path only, optional): NumPy copy of `bounds`; lets the library build the block
    table on the host (exact choice of the blocking plan, one small kernel less).  It must hold the same values as
    the device tensor whenever the batch runs - a plan that is re-run after `bounds` was overwritten on the device
    needs a new plan (or no `bounds_host`).
    `rirs` may be a RirBank (Renderer.rir_bank) of the same (P, C, L) instead of the raw RIRs, on every path."""
    dry: T.Any
    rirs: T.Any
    bounds: T.Any
    bounds_host: T.Any = None
    normalize_rirs: bool = False      # rirs = raw simulator output (formats.stack_rirs): divide by their global
                                      # abs-max on the device like generate_rir_combination (SonicSim_audio.py:398)
    direct_taps: int = 0              # > 0: also render the direct-path stem (every RIR row cut `direct_taps` taps
                                      # after its peak, see SS_DIRECT_TARGET) into the source's direct_outs entry
    window: T.Optional[T.Tuple[T.Any, int]] = None  # (start, length): render only output samples [start, start + length)
                                      # into a (C, length) output, bit-identical to those samples of the full render.
                                      # Device path: `start` may be a one-element CUDA int32 tensor (0-d, e.g.
                                      # starts[k]) read on the device at every run - a plan's crop can move between
                                      # runs without host work; out-of-range starts are clamped (check_device_errors)


class StaticSource(T.NamedTuple):
    """One static source: dry (N,), RIR (C, L), or a RirBank of shape (C, L) / (1, C, L)."""
    dry: T.Any
    rir: T.Any
    normalize_rirs: bool = False
    direct_taps: int = 0              # as MovingSource.direct_taps
    window: T.Optional[T.Tuple[T.Any, int]] = None  # as MovingSource.window


class Mixture(T.NamedTuple):
    """One training mixture of a device plan (Renderer.plan_device): the separation dataloader's (mix_wav, speaker_wav)
    (movingdatamodule.py:56-126) assembled on the device from the plan's own stems at every run.  `speakers` / `noises`:
    indices into the plan's `sources` (speaker 0 is the reference; 1 to 8 of each, each stem at most once per mixture,
    a stem may serve several mixtures), every stem of one (C, T).  `sirs`: CUDA float32 tensor of S - 1 elements (dB,
    e.g. sirs[b] of a (B, S - 1) tensor), None when S == 1; `snr`: one-element CUDA float32 tensor (dB, e.g. snr[b]);
    both are read on the device at every run.  Outputs, CUDA float32 and contiguous (slices of batch tensors such as
    mix[b] are the intended use): `mix` (C, T), or (T,) with `mono`; `speakers_out` (S, C, T) or (S, T): the speakers
    after their gains; `rms_db` (S,): compute_mch_rms_dB of every speaker stem before its gain (-200 for silence), for
    the dataloader's silence rule (redraw when a speaker is below -40 dB).  `mono`: fold every stem to its channel
    mean first (float32 sum in channel order, then a division by C).  `noise_delay`: overlap_audio's shift of the summed
    noise, in elements (see ss_mix_item).  `direct_out` (S, C, T) or (S, T), the dereverberation targets: each speaker's
    direct-path stem (the speaker's source needs direct_taps and a direct_outs entry) folded like the mixture's stems
    and scaled by that speaker's float32 gain with the multiply that gives speakers_out, so that target s is
    speakers_out[s] with the direct path in place of the reverberant stem (speaker 0: its folded direct stem).  The
    gains stay those of the reverberant crops, as the dataloader defines them."""
    speakers: T.Sequence[int]
    noises: T.Sequence[int]
    sirs: T.Any
    snr: T.Any
    mix: T.Any
    speakers_out: T.Any = None
    rms_db: T.Any = None
    mono: bool = False
    noise_delay: int = 0
    direct_out: T.Any = None


class _PooledFields(T.NamedTuple):
    pool: T.Any
    pick: T.Any
    window: T.Tuple[T.Any, int]
    direct_taps: int = 0
    dry: T.Any = None


class Pooled(_PooledFields):
    """A pooled slot of a device plan (Renderer.plan_device): at every run it renders the candidate of `pool`
    (Renderer.source_pool) named by `pick`, a one-element CUDA int32 tensor read on the device at that run (e.g.
    picks[b, k] of a (B, S) tensor) - the dataloader's random choice of scene, speakers and noise without host work.
    `window` = (start, length) as MovingSource.window: the start an int or a one-element CUDA int32 tensor; the length
    at most every candidate's N.  The output is (C, length).  `direct_taps` > 0 also renders the direct-path stem, which
    needs every candidate's bank to hold a direct set with these taps.  A pick outside [0, n) is clamped into range and a
    start beyond the picked candidate's N - length is clamped too (check_device_errors).  Only plan_device takes it.
    `dry`, a DryPick, makes it a dry-picked slot: the picked candidate renders with the dry signal the DryPick names in
    place of its own; a DryStream makes it a stream slot, whose dry signal is laid out from utterances at every run, and
    a BackgroundStream a bed slot, whose noise or music bed is laid out from clips at every run.  `trajectory`, a
    Trajectory, renders the picked candidate along the path and timing it holds at that run instead of the candidate's
    own.  It is a keyword attribute outside the tuple, as DryStream.lufs is: a Pooled stays the five-field tuple."""

    def __new__(cls, pool, pick, window, direct_taps=0, dry=None, trajectory=None):
        self = super().__new__(cls, pool, pick, window, direct_taps, dry)
        self.trajectory = trajectory
        return self

    def _replace(self, **kw):
        trajectory = kw.pop("trajectory", self.trajectory)
        return Pooled(*super()._replace(**kw), trajectory=trajectory)

    def __repr__(self):
        return "%s, trajectory=%r)" % (super().__repr__()[:-1], self.trajectory)

    def __getnewargs__(self):
        return tuple(self) + (self.trajectory,)


class Trajectory(T.NamedTuple):
    """The trajectory of a pooled slot (Pooled.trajectory) of a moving pool, read on the device at every run: `path` a
    contiguous 3-element CUDA int32 tensor (a, b, dir) with 0 <= a < b <= P - 1 of the picked candidate, dir 0 for the
    forward path over positions a, a + 1, ..., b or 1 for the reverse path b, b - 1, ..., a; `bounds` a contiguous CUDA
    int32 tensor of the pool's p_max entries (SourcePool.p_max, its largest P), whose first b - a + 1 are the visited
    path's cumulative segment bounds (0 first, the candidate's N last, non-decreasing; SonicSim_moving.bounds_from_counts
    of its per-segment sample counts).  The slot renders visited position j with the candidate's RIRs at position a + j
    (forward) or b - j (reverse) and these bounds; its dry signal, window, direct stem, dry pick, stream or bed stay as
    they are.  (0, P - 1, 0) with the candidate's own bounds renders bit for bit the slot without a trajectory.  An
    invalid path or bounds table renders the candidate's own forward path and bounds (check_device_errors raises
    ValueError).  Device pools only, without loudness gains or pair gains (both measured with the stored timing); a
    CropDraw speaker with a trajectory needs a DryPick or a DryStream, whose level tables do not depend on it.  A
    StemLoudness slot measures its whole stem with the run's trajectory."""
    path: T.Any
    bounds: T.Any


class DryPick(T.NamedTuple):
    """The dry signal of a pooled slot (Pooled.dry), picked on the device at every run independently of the slot's
    candidate: `pool` a DryPool (Renderer.dry_pool), `pick` a one-element CUDA int32 tensor (e.g. dry_picks[b, k] of a
    (B, S) tensor) naming one of its signals.  At every run the slot renders its picked candidate - RIRs, trajectory, N,
    blocking unchanged - with the first N samples of that signal as its dry signal, bit for bit what render_device gives
    for the candidate with that dry signal and the same window.  A pick outside [0, n) is clamped into range
    (check_device_errors raises IndexError).  Every signal of the pool must be at least as long as the slot pool's longest
    candidate; host pools take dry picks only from a host or a 16-bit dry pool.  In a CropDraw, a dry-picked speaker is
    tested on its dry crop, from the dry pool's level tables (dry_pool(..., levels=True)).  `gains`, a PairGains of the slot's pool and
    this dry pool (Renderer.pair_gains), stores the slot's stems at the picked pair's measured loudness gain, in place of
    the candidate's own; a pool with loudness gains takes only dry picks with `gains`."""
    pool: T.Any
    pick: T.Any
    gains: T.Any = None


class _DryStreamFields(T.NamedTuple):
    pool: T.Any
    ids: T.Any
    offsets: T.Any


class DryStream(_DryStreamFields):
    """The dry signal of a pooled slot (Pooled.dry) laid out at every run from utterances, as create_long_audio lays
    out a speech stream (SonicSim_audio.py:231-277): `pool` a 16-bit DryPool of n utterances (dry_pool(...,
    dtype="int16")), `ids` and `offsets` contiguous 1-D CUDA int32 tensors of equal length m, 1 <= m <= 128 (e.g. rows
    of (B, S, m) tensors from dry.long_audio_layouts), read on the device at every run.  The layout is walked in order:
    an entry with id < 0 is empty and skipped; one with id >= n, offset < 0 or offset before the end of the last kept
    entry is invalid and skipped (check_device_errors raises ValueError); any other places utterance `id` at samples
    [offset, offset + its length) of the stream.  The slot renders its picked candidate with the stream's first N
    samples, zeros where no utterance lies (an utterance reaching past N is cut there): bit for bit a DryPick from a
    16-bit pool holding the assembled stream.  A stream speaker of a CropDraw is tested on its crop's energy, summed per
    utterance from the pool's level tables (dry_pool(..., levels=True)).  Pools with loudness gains take no streams.
    `lufs`, a StemLoudness, stores the slot's crops at SonicSet's loudness, measured over the whole stem at every run.
    It is a keyword attribute outside the tuple: a DryStream stays the (pool, ids, offsets) tuple that callers unpack,
    compare and rebuild (_replace and repr carry `lufs`; tuple equality does not look at it)."""

    def __new__(cls, pool, ids, offsets, lufs=None):
        self = super().__new__(cls, pool, ids, offsets)
        self.lufs = lufs
        return self

    def _replace(self, **kw):
        lufs = kw.pop("lufs", self.lufs)
        return DryStream(*super()._replace(**kw), lufs=lufs)

    def __repr__(self):
        return "%s, lufs=%r)" % (super().__repr__()[:-1], self.lufs)

    def __getnewargs__(self):
        return tuple(self) + (self.lufs,)


class BackgroundStream(T.NamedTuple):
    """The dry signal of a pooled slot (Pooled.dry) laid out at every run from clips, as create_background_audio lays
    out a noise or music bed (SonicSim_audio.py:279-340): `pool` a DryPool of n clips, float32 or 16-bit (e.g. from
    dry.background_clips), and `ids`, `offsets`, `heads`, `counts` contiguous 1-D CUDA int32 tensors of one length m,
    1 <= m <= 128 (e.g. rows of (B, m) tensors from dry.background_audio_layouts), read on the device at every run.
    The layout is walked in order: an entry with id < 0 is empty and skipped; one with id >= n, offset < 0, head < 0,
    count < 1, head + count beyond the clip, or an offset before the end of the last kept entry is invalid and skipped
    (check_device_errors raises ValueError); any other places clip samples [head, head + count) at stream samples
    [offset, offset + count).  The slot renders its picked candidate with the stream's first N samples, zeros where no
    clip lies: bit for bit a DryPick from a pool of the same dtype holding the assembled bed.  A bed slot may read a
    CropDraw's start but is none of its speakers; pools with loudness gains take no beds.  `lufs`, a StemLoudness,
    stores the slot's crops at SonicSet's loudness, measured over the whole stem at every run."""
    pool: T.Any
    ids: T.Any
    offsets: T.Any
    heads: T.Any
    counts: T.Any
    lufs: T.Any = None


class StemLoudness(T.NamedTuple):
    """The loudness target of a stream or bed slot (DryStream.lufs, BackgroundStream.lufs): SonicSet stores every stem
    loudness-normalised over the whole stem (SonicSet.py:97-101, get_lufs_norm_audio), and a stream or bed laid out at
    every run has no fixed stem to measure once.  At every run the plan renders the slot's whole stem [0, N), measures
    it like render_host(..., lufs_targets=) and stores the slot's crop, and its direct-path crop, cut out of that stem and
    scaled by the gain: bit for bit the crop at the run's start of render_host(..., lufs_targets=[target]) of the
    picked candidate with the stream or bed that run lays out.  `target`: a one-element CUDA float64 tensor read at
    every run (e.g. lufs[b, k] of a (B, K) tensor refreshed with uniform_(-19, -15) before run()); a non-finite target
    stores the slot unscaled (check_device_errors raises ValueError).  `result`: None, or a contiguous two-element CUDA
    float64 tensor that receives (measured LUFS, linear gain) at every run (gain NaN for a non-finite target).  `sr`:
    the rate of the gating plan, built once from the pool's N.  The slot's SourcePool must be device-resident, without
    loudness gains, with C <= 8 and every candidate of one N (SonicSet's stems are all 60 s); every loudness slot of a
    plan has one sr.  Each slot adds C * N floats of plan scratch (twice that with direct_taps) and 20 * C doubles
    per 0.1 s of its N; a plan with such slots launches 7 kernels more per run, plus a launch group per further chunk its
    whole stems take."""
    target: T.Any
    result: T.Any = None
    sr: float = 16000.0


class _LayoutDrawFields(T.NamedTuple):
    slot: int
    rng: T.Any
    total: int
    sample_rate: int = 16000
    select_lengths: T.Any = None


class LayoutDraw(_LayoutDrawFields):
    """A stream or bed slot whose layout the plan draws itself at every run (Renderer.plan_device(layouts=...)), by the
    rule of dry.long_audio_layouts (a DryStream slot) or dry.background_audio_layouts (a BackgroundStream slot), in one
    kernel launch at the head of the run.  `slot`: index into the plan's sources.  `rng`: a two-element CUDA int64 tensor
    (seed, t) read at every run and never written (one tensor may serve every draw of a plan): the same (seed, t) draws
    the same layouts bit for bit, and a training step bumps t (rng[1] += 1) before plan.run(), as u.uniform_() refreshes
    a CropDraw.  Draw r of `layouts` takes Philox4x32-10 blocks (b, r, t) under the key seed (include/sonicsim_b200.h,
    ss_layout_draw, states the stream).  `total`: the samples of the stream create_long_audio or create_background_audio
    would build; gaps and tails are uniform in {0, ..., 10 * sample_rate}.  `select_lengths` (bed slots only): n
    non-negative selection lengths, e.g. the clips' native-rate lengths from SonicSet's JSON (see
    dry.background_audio_layouts); None selects by the clip lengths.  The draw writes the slot's own ids, offsets (and
    heads, counts) tensors, which then hold that run's layout.  The layouts match the rules in distribution, not torch's
    bits.  A row may select at most 1024 utterances or clips (dry.long_audio_max_selected,
    dry.background_audio_max_selected).

    Speaker groups (stream slots only), as SonicSet builds every stream from one LibriSpeech speaker: `groups`, G + 1
    host bounds 0 = groups[0] < ... < groups[G] = the pool's n (a sequence, array or tensor; dry.speaker_groups builds
    them), splits the utterance pool into G contiguous groups, and `group`, a one-element CUDA int32 tensor read at
    every run (e.g. spk[b, k] of a (B, S) tensor a ValueDraw(spk, rng, 0, G, distinct=True) writes), names the group
    this run lays the stream out from.  The row is then exactly the ungrouped draw over a pool of that group's
    utterances alone, with the same words, its ids shifted by groups[g] into the whole pool; a group outside [0, G) is
    clamped into range (check_device_errors raises IndexError).  Give both or neither; 1024 bounds every group's
    selection (dry.long_audio_max_selected(lengths, total, groups)).  `groups` and `group` are attributes outside the
    tuple: a LayoutDraw stays the (slot, rng, total, sample_rate, select_lengths) tuple callers unpack and rebuild
    (_replace and repr carry them; tuple equality does not look at them)."""

    def __new__(cls, slot, rng, total, sample_rate=16000, select_lengths=None, groups=None, group=None):
        self = super().__new__(cls, slot, rng, total, sample_rate, select_lengths)
        self.groups, self.group = groups, group
        return self

    def _replace(self, **kw):
        groups, group = kw.pop("groups", self.groups), kw.pop("group", self.group)
        return LayoutDraw(*super()._replace(**kw), groups=groups, group=group)

    def __repr__(self):
        return "%s, groups=%r, group=%r)" % (super().__repr__()[:-1], self.groups, self.group)

    def __getnewargs__(self):
        return tuple(self) + (self.groups, self.group)


class ValueDraw(T.NamedTuple):
    """Per-run values that a device plan draws itself at the head of every run (Renderer.plan_device(values=...)), in
    one kernel launch before everything that reads them: the picks, dry picks, crop starts, SIRs, SNRs, CropDraw
    variates and StemLoudness targets that a training loop would otherwise refresh with torch before plan.run().
    `out`: a contiguous CUDA tensor of shape (B,) or (B, k), 1 <= k <= 4096, written at every run; the plan's other
    parts read it as they read any such tensor.  float32 / float64: uniform reals in [low, high) (float32 bounds must be
    exact in float32); int32: uniform integers in [low, high).  `rng`: a two-element CUDA int64 tensor (seed, t) read at
    every run and never written, as LayoutDraw.rng (one tensor may serve every draw): a training step is then

        rng[1] += 1
        plan.run()

    and the batch is a pure function of (seed, t).  `distinct` (int32 only, k <= min(64, high - low)): each row is an
    ordered sample without replacement, as random.sample(range(low, high), k).  `base` (int32 only): the `out`, of shape
    (B,), of an earlier int32 ValueDraw of the same plan; the values become base[b] * stride + value (stride >= 1), e.g.
    speaker picks within the scene a first draw chose, over scene-major pools.  Draw r of `values` takes Philox4x32-10
    blocks under the key seed in a stream of its own (include/sonicsim_b200.h, ss_value_draw, states it), apart from
    the layout draws' blocks.  Every ValueDraw of a plan has the same B, at most 65535.  The values match the rules in
    distribution, not torch's or `random`'s bits."""
    out: T.Any
    rng: T.Any
    low: float = 0.0
    high: float = 1.0
    distinct: bool = False
    base: T.Any = None
    stride: int = 0


class CropDraw(T.NamedTuple):
    """A crop start drawn on the device at every run of a device plan (Renderer.plan_device(draws=...)): the dataloader's
    start loop (movingdatamodule.py:81-99).  `start`: the one-element CUDA int32 tensor that the windows of this
    example's pooled slots use as their start (those slots are the draw's readers, all of one window length).  `speakers`:
    indices into the plan's sources, 1 to 8 pooled slots among the readers whose pools have level tables
    (Renderer.source_pool(levels=...)).  `u`: a CUDA float64 tensor of 1 to 4096 uniform variates in [0, 1) (e.g. a row
    of torch.rand((B, 101), dtype=torch.float64)), read at every run.  Try t starts at min(floor(u[t] * M), M - 1), M
    the number of starts every reader's picked candidate holds; the draw keeps the first try at which no speaker's crop is
    below `threshold_db` (compute_mch_rms_dB of the crop), else the last try.  `used`, if given (one-element CUDA int32),
    receives the 1-based index of the kept try, or 0 when every try was silent."""
    start: T.Any
    speakers: T.Sequence[int]
    u: T.Any
    used: T.Any = None
    threshold_db: float = -40.0


LEVELS = {None: None, "mono": _lib.SS_MIX_MONO, "channels": 0}


def _is_tensor(v) -> bool:
    return type(v).__module__.split(".")[0] == "torch"


def _tensor(t, api, owner, field, dtype, device, shape=None, count=None):
    """Checks a tensor argument before any C call and returns its data_ptr(): a contiguous `dtype` CUDA tensor on
    cuda:`device`, of `count` = (lo, hi) elements and of shape `shape` (a str entry such as "C" takes any size) when
    given.  `owner` ("source 3", "mixture 1", ...) names what holds the tensor; None for an argument of `api` itself."""
    import torch
    what = "%s: %s" % (api, field) if owner is None else "%s: %s of %s" % (api, field, owner)
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor on cuda:%d" % (what, device))
    if t.device.index != device:
        raise ValueError("%s is on cuda:%s, the renderer on cuda:%d" % (what, t.device.index, device))
    if t.dtype != dtype:
        raise ValueError("%s must be %s, got %s" % (what, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % what)
    if count is not None and not count[0] <= t.numel() <= count[1]:
        lo, hi = count
        raise ValueError("%s must hold %s element%s, got %d" % (what, lo if lo == hi else "%d to %d" % count,
                                                                  "" if hi == 1 else "s", t.numel()))
    if shape is not None and (t.dim() != len(shape) or
                              any(w != g for w, g in zip(shape, t.shape) if not isinstance(w, str))):
        raise ValueError("%s must have shape %s, got %s" % (what, str(tuple(shape)).replace("'", ""), tuple(t.shape)))
    return t.data_ptr()


def _bounds(b, P, what, keep):
    """A host bounds table as a contiguous int32 array of P entries, kept alive in `keep`; `what` names it."""
    a = np.ascontiguousarray(b, dtype=np.int32)
    if a.shape != (P,):
        raise ValueError("%s must have P = %d entries, got shape %s" % (what, P, a.shape))
    keep.append(a)
    return a


def _window(s, i, N):
    """(win_start, win_len, samples per output row) of source i; a window must lie inside [0, N] and not be empty."""
    if s.window is None:
        return 0, 0, N
    if _is_tensor(s.window[0]):
        raise ValueError("window of source %d: a tensor start is read on the device at every run; only render_device "
                         "and plan_device take one" % i)
    a, n = (int(v) for v in s.window)
    if a < 0 or n < 1 or a + n > N:
        raise ValueError("window of source %d must be (start, length) with 0 <= start, length >= 1 and "
                         "start + length <= N = %d, got (%d, %d)" % (i, N, a, n))
    return a, n, n


def _window_dev(s, i, N, device):
    """_window for the device path, plus the start tensor of a moving window (else None): a one-element CUDA int32
    tensor on cuda:`device`, whose value the kernels read at every run (win_start_dev)."""
    if s.window is None or not _is_tensor(s.window[0]):
        return _window(s, i, N) + (None,)
    import torch
    t, n = s.window[0], int(s.window[1])
    if t.dtype != torch.int32 or t.numel() != 1:
        raise ValueError("window of source %d: a start tensor must hold one int32, got %s with %d elements"
                         % (i, t.dtype, t.numel()))
    if not t.is_cuda or t.device.index != device:
        raise ValueError("window of source %d: a start tensor must be on cuda:%d, got %s" % (i, device, t.device))
    if n < 1 or n > N:
        raise ValueError("window of source %d must have 1 <= length <= N = %d, got %d" % (i, N, n))
    return 0, n, n, t


def _flags(s, i, direct_out) -> int:
    """ss_source.flags of source i; checks that a direct-path stem has an output and an output has a stem."""
    taps = int(s.direct_taps)
    if taps < 0:
        raise ValueError("direct_taps of source %d must be >= 0, got %d" % (i, taps))
    if taps > 0 and direct_out is None:
        raise ValueError("source %d has direct_taps = %d but no direct output (direct_outs[%d])" % (i, taps, i))
    if taps == 0 and direct_out is not None:
        raise ValueError("direct_outs[%d] is given but source %d has no direct_taps" % (i, i))
    norm = getattr(s, "normalize_rirs", False)              # (a pooled slot has none: normalisation is the banks')
    return (_lib.SS_RIR_NORMALIZE if norm else 0) | (_lib.SS_DIRECT_TARGET if taps > 0 else 0)


class _Held:
    """Device memory that plans (and pools) hold: close() refuses it to new users and frees it once no holder is left."""
    _closing, _plans = False, 0

    @property
    def closed(self) -> bool:
        """True once close() was called: new sources may not use it (plans made before keep working)."""
        return self._closing or not self._h

    def close(self):
        """Refuse it to new sources and free its device memory - at once, or, while plans that use it are alive, when
        the last of them is closed or collected (their runs keep reading it until then)."""
        self._closing = True
        if self._plans == 0:
            self._free()

    def _hold(self):
        self._plans += 1

    def _release(self):
        self._plans -= 1
        if self._closing and self._plans == 0:
            self._free()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class RirBank(_Held):
    """The half spectra of one RIR set, transformed once and held in device memory (Renderer.rir_bank; ss_bank of the C
    ABI).  Pass it as `MovingSource.rirs` / `StaticSource.rir`: the source renders bit-identically to the same source
    given the raw RIRs, which are never read again.  It belongs to the context of the renderer that made it.  Every
    render that uses it is ordered after its construction by the library, on every path, whatever stream built it.
    Plans and source pools hold the bank: it is freed only once it is closed (or collected) and nothing alive uses it.
    A host bank (`host` True, Renderer.rir_bank(..., host=True)) holds its spectra in pinned host memory
    (`host_nbytes`; `nbytes` counts device bytes only) and serves only as a candidate of a host source pool.  `form` is
    "spectra", or "taps" for a tap-form host bank (SS_BANK_TAPS), which holds the (normalised) taps in rows of 4096
    instead, half the pinned bytes, and whose pools transform the rows each run stages on the device."""

    def __init__(self, renderer, handle, shape, normalize, direct_taps, host=False, form="spectra"):
        self.renderer, self._h = renderer, handle
        self.shape = tuple(int(v) for v in shape)          # as given: (P, C, L) or (C, L)
        self.normalize, self.direct_taps, self.host = bool(normalize), int(direct_taps), bool(host)
        self.form = form
        self.nbytes = int(renderer.lib.ss_bank_bytes(handle))
        self.host_nbytes = int(renderer.lib.ss_bank_host_bytes(handle))

    @property
    def pcl(self) -> T.Tuple[int, int, int]:
        return self.shape if len(self.shape) == 3 else (1,) + self.shape

    def _free(self):
        if self._h:
            self.renderer.lib.ss_bank_destroy(self._h)
            self._h = ctypes.c_void_p()


class SourcePool(_Held):
    """A set of banked candidate sources validated and uploaded once (Renderer.source_pool; ss_pool of the C ABI), which
    pooled slots (render.Pooled) of device plans pick from at every run.  `n` candidates of one `mode` and `C`; `L` is
    the longest candidate's RIR length (candidates may differ in L, each keeps its own bank); `n_min` is the shortest candidate's N (the longest window a slot may take); `direct_taps` > 0 when every candidate's
    bank holds a direct set with these taps.  The pool holds its candidates' banks and keeps their tensors alive; plans
    hold the pool, which is freed once it is closed (or collected) and no live plan uses it any more.  `levels` is None,
    "mono" or "channels": the level tables the pool holds for start draws (CropDraw), included in `nbytes`.
    `loudness` is an (n, 2) float64 array of every candidate's measured integrated loudness (LUFS) and linear gain
    (ss_pool_loudness), NaN for a candidate without a target; `nbytes` includes the gains (4 bytes per candidate), and
    the candidates' partition counts (4 bytes per candidate) when their K = ceil(L / 4096) differ (ss_pool_bytes).
    `resident` is "device", or "host" for a pool over host banks (RirBank.host): its dry signals, banks and level tables
    stay in pinned host memory (`host_nbytes`, banks not included), `nbytes` counts its device bytes, and every plan run
    copies only what its slots read (ss_pool_host_bytes, INTEGRATION.md)."""

    def __init__(self, renderer, handle, candidates, mode, C, L, n_min, direct_taps, levels=None, loudness=None,
                 sizes=None, resident="device", gains=False):
        self.renderer, self._h = renderer, handle
        self.gains = bool(gains)                           # loudness gains (lufs_targets): no dry picks
        self.candidates = list(candidates)
        self.resident = resident
        self._sizes = list(sizes) if sizes is not None else [int(s.dry.numel()) for s in self.candidates]
        self.host_nbytes = int(renderer.lib.ss_pool_host_bytes(handle))
        self.n, self.mode, self.C, self.L = len(self.candidates), mode, C, L
        self.p_max = max(_rirs(c)[2] for c in self.candidates)     # the most positions: a Trajectory's bounds length
        self.n_min, self.direct_taps, self.levels = n_min, direct_taps, levels
        self._loudness = loudness if loudness is not None else np.full((self.n, 2), np.nan)
        self.nbytes = int(renderer.lib.ss_pool_bytes(handle))
        self._banks = _hold_banks(self, self.candidates)

    @property
    def loudness(self) -> np.ndarray:
        """(n, 2) float64: measured LUFS and linear gain of every candidate (ss_pool_loudness), NaN when unmeasured."""
        return self._loudness.copy()

    def level_table(self, i):
        """A float64 CUDA copy of candidate i's level table (N + 1 values: Q[0] = 0, Q[n + 1] = Q[n] + e[n]), see
        ss_pool_levels; None without tables."""
        import torch
        if self.closed or self.levels is None or not 0 <= i < self.n:
            return None
        ptr = self.renderer.lib.ss_pool_level_table(self._h, int(i))
        n = self._sizes[i] + 1
        if self.resident == "host":                        # pinned, mapped host memory: copied from the host side
            host = np.ctypeslib.as_array((ctypes.c_double * n).from_address(ptr))
            return torch.from_numpy(host.copy()).to("cuda:%d" % self.renderer.device)

        class _View:
            __cuda_array_interface__ = {"shape": (n,), "typestr": "<f8", "data": (ptr, False), "version": 3}
        with torch.cuda.device(self.renderer.device):
            return torch.as_tensor(_View(), device="cuda:%d" % self.renderer.device).clone()

    def _free(self):
        if self._h:
            self.renderer.lib.ss_pool_destroy(self._h)
            self._h = ctypes.c_void_p()
            self._banks()                      # the pool no longer reads its banks


class DryPool(_Held):
    """A set of `n` dry signals (Renderer.dry_pool; ss_dry_pool of the C ABI), which dry-picked
    slots (DryPick) take their dry signal from at every run.  `sizes` are the signals' lengths and `n_min` the shortest:
    the longest candidate N a pool of slots that pick from it may have.  With `levels` True it holds every signal's level
    table (float64 prefix sums of its squares, 8 bytes per sample, in `nbytes`), which CropDraw reads for dry-picked
    speakers.  A device dry pool (`resident` "device") references the signals' tensors (`signals`) and keeps them alive;
    a host dry pool (`resident` "host") copied them into pinned host memory, where its level tables also stay
    (`host_nbytes`; `nbytes` then counts only its pointer arrays), and every plan run copies only the samples its slots
    read (ss_dry_pool_host_bytes, INTEGRATION.md).  A 16-bit pool (`dtype` "int16") holds every signal as its int16
    samples k, standing for k / 32768, in an arena it owns (2 bytes per sample), and its level tables at `level_stride`
    64 (one float64 per 64 samples); it behaves bit for bit as the float32 pool of the same values.  Plans hold the
    pool, which is freed once it is closed (or collected) and no live plan uses it."""
    resident = "device"
    dtype = "float32"

    def __init__(self, renderer, handle, signals, sizes, levels, resident="device", dtype="float32"):
        self.renderer, self._h = renderer, handle
        self.signals = list(signals)
        self.sizes = [int(v) for v in sizes]
        self.n, self.levels, self.resident, self.dtype = len(self.sizes), bool(levels), resident, dtype
        self.n_min = min(self.sizes)
        self.nbytes = int(renderer.lib.ss_dry_pool_bytes(handle))
        self.host_nbytes = int(renderer.lib.ss_dry_pool_host_bytes(handle))
        self.level_stride = int(renderer.lib.ss_dry_pool_level_stride(handle))

    def _read(self, ptr, n, typestr, ctype):
        """A NumPy copy of n elements at `ptr`, in this pool's residency (a host address for a host pool)."""
        import torch
        if self.resident == "host":                        # pinned, mapped host memory: copied from the host side
            return np.ctypeslib.as_array((ctype * n).from_address(ptr)).copy()

        class _View:
            __cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}
        with torch.cuda.device(self.renderer.device):
            return torch.as_tensor(_View(), device="cuda:%d" % self.renderer.device).cpu().numpy()

    def level_table(self, i):
        """A float64 CUDA copy of signal i's level table (N + 1 values: Q[0] = 0, Q[n + 1] = Q[n] + x[n]^2), or None
        without tables.  A 16-bit pool's is rebuilt on the host from its sparse table and the signal's samples, bit for
        bit the float32 pool's (_levels_from_sparse)."""
        import torch
        if self.closed or not self.levels or not 0 <= i < self.n:
            return None
        lib, N = self.renderer.lib, self.sizes[i]
        ptr = lib.ss_dry_pool_level_table(self._h, int(i))
        if self.dtype == "int16":
            q = self._read(ptr, -(-N // self.level_stride) + 1, "<f8", ctypes.c_double)
            x = self._read(lib.ss_dry_pool_signal_i16(self._h, int(i)), N, "<i2", ctypes.c_int16)
            return torch.from_numpy(_levels_from_sparse(q, x)).to("cuda:%d" % self.renderer.device)
        if self.resident == "host":
            return torch.from_numpy(self._read(ptr, N + 1, "<f8", ctypes.c_double)).to("cuda:%d" % self.renderer.device)

        class _View:
            __cuda_array_interface__ = {"shape": (N + 1,), "typestr": "<f8", "data": (ptr, False), "version": 3}
        with torch.cuda.device(self.renderer.device):
            return torch.as_tensor(_View(), device="cuda:%d" % self.renderer.device).clone()

    def _free(self):
        if self._h:
            self.renderer.lib.ss_dry_pool_destroy(self._h)
            self._h = ctypes.c_void_p()


class PairGains(_Held):
    """The loudness gain of every (dry signal, candidate) pair of a SourcePool and a DryPool (Renderer.pair_gains;
    ss_pair_gains of the C ABI), which dry-picked slots (DryPick(..., gains=)) store their stems with.  `loudness` is an
    (n_dry, n, 2) float64 array of every pair's measured integrated loudness (LUFS) and linear gain, NaN for a pair
    without a target; `nbytes` counts its device bytes (4 per pair).  Plans hold it: it is freed once it is closed (or
    collected) and no live plan uses it."""

    def __init__(self, renderer, handle, pool, dry_pool, loudness):
        self.renderer, self._h = renderer, handle
        self.pool, self.dry_pool = pool, dry_pool
        self._loudness = loudness
        self.nbytes = int(renderer.lib.ss_pair_gains_bytes(handle))

    @property
    def loudness(self) -> np.ndarray:
        """(n_dry, n, 2) float64: measured LUFS and linear gain of pair (d, i), NaN when unmeasured."""
        return self._loudness.copy()

    def _free(self):
        if self._h:
            self.renderer.lib.ss_pair_gains_destroy(self._h)
            self._h = ctypes.c_void_p()


def _rirs(s, conv=None):
    """Where a MovingSource / StaticSource takes its RIRs from: (RirBank or None, raw RIRs or None, P, C, L, mode).
    Raw RIRs go through conv(raw, field name, shape), the caller's conversion or check, and their shape is read from
    what it returns (a NumPy array or a tensor); without `conv` they are returned as given, with P, C, L None."""
    static = isinstance(s, StaticSource)
    r, mode = (s.rir, _lib.SS_STATIC) if static else (s.rirs, _lib.SS_MOVING_BOUNDS)
    if isinstance(r, RirBank):
        return (r, None) + ((1,) + r.pcl[1:] if static else r.pcl) + (mode,)
    if conv is None:
        return None, r, None, None, None, mode
    if static:
        r = conv(r, "rir", ("C", "L"))
        (C, L), P = r.shape, 1
    else:
        r = conv(r, "rirs", ("P", "C", "L"))
        P, C, L = r.shape
    return None, r, P, C, L, mode


def _pool_host_dry(dry, api, own, device, keep):
    """(pointer, N) of a dry signal that a host pool (a candidate's) or a host dry pool copies (`api` names the call):
    a CUDA float32 tensor of the renderer's device, or a 1-D NumPy array / CPU tensor (converted to contiguous float32,
    kept alive in `keep`)."""
    if _is_tensor(dry) and dry.is_cuda:
        import torch
        return _tensor(dry, api, own, "dry", torch.float32, device), dry.numel()
    a = np.ascontiguousarray(dry.numpy() if _is_tensor(dry) else dry, dtype=np.float32)
    if a.ndim != 1 or a.size < 1:
        raise ValueError("%s: dry of %s must be 1-D and not empty, got shape %s" % (api, own, a.shape))
    keep.append(a)
    return a.ctypes.data, a.size


I16_MAX_SAMPLES = 1 << 23                  # a 16-bit dry signal's longest (ss_dry_pool_create_i16)
I16_STRIDE = 64                            # its level tables' stride


def _levels_from_sparse(q, x):
    """The full level table (N + 1 float64) of a 16-bit signal x (N int16 samples, k standing for k / 32768) from its
    sparse table q (q[j] = Q[min(64 j, N)]): Q[s] = q[s // 64] plus the float64 sum of the float32 squares of samples
    [64 (s // 64), s).  Every partial sum is a multiple of 2^-30 below 2^23, exact in float64, so the result is the
    float32 pool's table bit for bit whatever the order of the sums."""
    N = x.size
    m = -(-N // I16_STRIDE)
    v = x.astype(np.float32) * np.float32(1.0 / 32768.0)
    sq = np.zeros(m * I16_STRIDE, np.float64)
    sq[:N] = (v * v).astype(np.float64)                # the float32 square k_levels adds
    blocks = sq.reshape(m, I16_STRIDE)
    part = np.cumsum(blocks, axis=1) - blocks          # exclusive, within each block
    Q = np.empty(N + 1, np.float64)
    Q[:N] = (q[:m, None] + part).reshape(-1)[:N]
    Q[N] = q[m]
    return Q


def _as_i16(x, own, device, keep):
    """(pointer, N) of a signal for a 16-bit dry pool: an int16 NumPy array or CPU / CUDA tensor, or a float one whose
    every sample is exactly k / 32768 with -32768 <= k <= 32767 (converted; the first sample off that grid is named).
    Anything else - other dtypes, a sample off the grid or +1.0, an empty or longer than 2^23 signal - is a ValueError.
    Converted or host arrays are kept alive in `keep`; a CUDA tensor must be on cuda:`device`."""
    tensor = _is_tensor(x)
    cuda = tensor and x.is_cuda
    if cuda and x.device.index != device:
        raise ValueError("dry_pool: %s is on cuda:%s, the renderer on cuda:%d" % (own, x.device.index, device))
    a = x if cuda else x.numpy() if tensor else np.asarray(x)
    if a.ndim != 1 or a.shape[0] < 1 or a.shape[0] > I16_MAX_SAMPLES:
        raise ValueError("dry_pool: %s must be 1-D with 1 to 2^23 samples for dtype int16, got shape %s"
                         % (own, tuple(a.shape)))
    if cuda:
        import torch
        if a.dtype == torch.int16:
            a = a.contiguous()
        elif a.dtype.is_floating_point:
            k = a.double() * 32768.0
            bad = ~((k == torch.floor(k)) & (k >= -32768.0) & (k <= 32767.0))   # (NaN and inf fail too)
            if bool(bad.any()):
                j = int(torch.nonzero(bad)[0, 0])
                raise ValueError("dry_pool: %s has sample %d = %r, not k / 32768 with k an int16"
                                 % (own, j, float(a[j])))
            a = k.to(torch.int16)
        else:
            raise ValueError("dry_pool: %s must be int16 or float on the int16 grid, got %s" % (own, a.dtype))
        keep.append(a)
        return a.data_ptr(), a.numel()
    if a.dtype == np.int16:
        a = np.ascontiguousarray(a)
    elif np.issubdtype(a.dtype, np.floating):
        k = a.astype(np.float64) * 32768.0
        with np.errstate(invalid="ignore"):
            bad = ~((k == np.floor(k)) & (k >= -32768.0) & (k <= 32767.0))
        if bad.any():
            j = int(np.argmax(bad))
            raise ValueError("dry_pool: %s has sample %d = %r, not k / 32768 with k an int16" % (own, j, float(a[j])))
        a = k.astype(np.int16)
    else:
        raise ValueError("dry_pool: %s must be int16 or float on the int16 grid, got %s" % (own, a.dtype))
    keep.append(a)
    return a.ctypes.data, a.size


def _cuda_tensors(obj):
    """Every CUDA tensor in `obj`, a nesting of tuples (NamedTuples included) and lists."""
    if _is_tensor(obj):
        return [obj] if obj.is_cuda else []
    if isinstance(obj, (tuple, list)):
        return [t for v in obj for t in _cuda_tensors(v)]
    return []


def _check_usable(held, renderer, what):
    """Refuses a closed RirBank / SourcePool, or one of another renderer's context; `what` names it."""
    if held.closed:
        raise ValueError("%s is closed" % what)
    if held.renderer.ctx.value != renderer.ctx.value:
        raise ValueError("%s belongs to another renderer's context" % what)


def _bank_of(renderer, s, i, P, C, L):
    """Checks a banked source against its bank before any C call; returns the ss_bank handle."""
    b = _rirs(s)[0]
    _check_usable(b, renderer, "source %d: its RirBank" % i)
    if b.pcl != (P, C, L):
        raise ValueError("source %d: its RirBank holds (P, C, L) = %s, the source has %s" % (i, b.pcl, (P, C, L)))
    if s.normalize_rirs:
        raise ValueError("source %d: normalisation is a property of its RirBank (normalize=%s); leave normalize_rirs "
                         "False" % (i, b.normalize))
    if getattr(b, "host", False):
        raise ValueError("source %d: its RirBank is a host bank (host=True), which serves only as a candidate of a "
                         "source pool" % i)
    if int(s.direct_taps) not in (0, b.direct_taps):
        raise ValueError("source %d: direct_taps = %d, its RirBank holds %s" % (
            i, int(s.direct_taps), "direct_taps = %d" % b.direct_taps if b.direct_taps else "no direct set"))
    return b._h.value


def _kind(k):
    return ("static" if k[0] == _lib.SS_STATIC else "moving", k[1])


def _refuse_pooled(sources, where):
    for i, s in enumerate(sources):
        if isinstance(s, Pooled):
            raise ValueError("%s: source %d is a pooled slot (render.Pooled), which only device plans (plan_device) "
                             "render" % (where, i))


def _release_banks(banks):
    for b in banks:
        b._release()


def _hold_banks(plan, sources):
    """The RirBanks and SourcePools of a plan's sources (of a pool's candidates) are held until the plan (the pool) is
    closed or collected: one closed meanwhile is freed only then.  Returns the finalizer that releases them (calling it
    releases them at once, once)."""
    banks = []
    for s in sources:
        # a dry-picked slot's dry pool and pair gains, a stream slot's utterance pool, a bed slot's clip pool
        dry = s.dry if isinstance(s, Pooled) and isinstance(s.dry, (DryPick, DryStream, BackgroundStream)) else None
        held = ([s.pool] + ([dry.pool, getattr(dry, "gains", None)] if dry else []) if isinstance(s, Pooled)
                else [_rirs(s)[0]])
        for b in held:
            if isinstance(b, (RirBank, SourcePool, DryPool, PairGains)) and all(b is not o for o in banks):
                banks.append(b)
    for b in banks:
        b._hold()
    return weakref.finalize(plan, _release_banks, banks)


def _check_direct_outs(direct_outs, n):
    if direct_outs is not None and len(direct_outs) != n:
        raise ValueError("%d sources but %d entries in direct_outs" % (n, len(direct_outs)))
    return direct_outs if direct_outs is not None else [None] * n


def _check_lufs(api, what, targets, n, sr):
    """Refuses, before any C call, loudness targets (when given) other than one finite value or None for each of the n
    stems, and sr <= 0; `what` names a stem ("source", "candidate")."""
    if targets is None:
        return
    if len(targets) != n:
        raise ValueError("%s: %d %ss but %d entries in lufs_targets" % (api, n, what, len(targets)))
    for i, t in enumerate(targets):
        if t is not None and not math.isfinite(float(t)):
            raise ValueError("%s: the loudness target of %s %d is not finite: %r" % (api, what, i, t))
    if not float(sr) > 0:
        raise ValueError("%s: sr must be > 0, got %r" % (api, sr))


def _post_lufs(targets, items, sr, results, keep):
    """The ss_post_lufs array of checked targets for the SsSource `items` (None without targets): stem i is measured
    like SonicSim_audio.lufs_norm into results[i].  The gating plans it points into, one per length, go to `keep`."""
    if targets is None:
        return None
    from .SonicSim_audio import gating_block_size, gating_plan
    post = (SsPostLufs * len(targets))()
    plans = {}
    for i, t in enumerate(targets):
        if t is None:
            continue
        N = items[i].N
        block = float(gating_block_size(N, sr))
        if N not in plans:
            plans[N] = gating_plan(N, float(sr), block)
        brk, blo, bhi = plans[N]
        post[i] = SsPostLufs(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data, n_e=len(brk) - 1,
                             n_blocks=len(blo), rate=float(sr), block_size=block, target_lufs=float(t),
                             result=results[i].ctypes.data)
    keep.append(plans)
    return post


class Renderer:
    """Owns the per-device ss_ctx.  One process per GPU (LOCAL_RANK picks the device by default)."""

    def __init__(self, device: T.Optional[int] = None):
        self.lib = _lib.load()
        self.device = _lib.default_device() if device is None else int(device)
        self.ctx = _lib.context(self.device)

    # ------------------------------------------------------------------ RIR spectrum banks
    def rir_bank(self, rirs, normalize: bool = False, direct_taps: int = 0, host: bool = False,
                 form: str = "spectra") -> RirBank:
        """Transform an RIR set (P, C, L) - or (C, L) for a static source - once into a RirBank on this renderer's
        device: a NumPy array is copied in and the call returns when the bank is complete; a CUDA float32 tensor of this
        device is transformed asynchronously on the current stream (keep it unchanged until that stream gets there).
        Either way the bank can be used at once, on every path: every render that uses it - render_host / plan_host on
        the library's own streams, render_device / plan_device on any stream - waits for its construction first.
        `normalize` / `direct_taps` are the normalize_rirs / direct_taps every source of the bank renders with (a bank
        with a direct set also serves sources with direct_taps = 0).  `host` moves the transformed bank into pinned host
        memory (SS_BANK_HOST; bit-identical spectra, the call returns once it is there): such a bank is only a candidate
        of a host source pool (source_pool), whose plans copy the rows each run reads to the device.  `form` = "taps"
        (host banks only, SS_BANK_TAPS) keeps the taps instead of their spectra - zero-padded rows of 4096, divided by the
        abs-max with `normalize` - at half the pinned bytes, a quarter with a direct set; its pools copy half the RIR
        bytes per run and transform them on the device, with the bits of a spectral host bank of the same RIRs."""
        taps = int(direct_taps)
        if taps < 0:
            raise ValueError("direct_taps must be >= 0, got %d" % taps)
        if form not in ("spectra", "taps"):
            raise ValueError("rir_bank: form must be 'spectra' or 'taps', got %r" % (form,))
        if form == "taps" and not host:
            raise ValueError("rir_bank: form='taps' is a host bank form: it needs host=True")
        flags = (_lib.SS_RIR_NORMALIZE if normalize else 0) | (_lib.SS_DIRECT_TARGET if taps > 0 else 0) | \
            (_lib.SS_BANK_HOST if host else 0) | (_lib.SS_BANK_TAPS if form == "taps" else 0)
        h = ctypes.c_void_p()
        dev = _is_tensor(rirs)
        if dev:
            import torch
            _tensor(rirs, "rir_bank", None, "rirs", torch.float32, self.device)
        a = rirs if dev else _as_f32(rirs)
        shape = tuple(a.shape)
        if len(shape) not in (2, 3):
            raise ValueError("rir_bank: rirs must be (P, C, L) or (C, L), got shape %s" % (shape,))
        P, C, L = shape if len(shape) == 3 else (1,) + shape
        if dev:
            stream = torch.cuda.current_stream(rirs.device).cuda_stream
            _lib.check(self.lib.ss_bank_create_dev(self.ctx, rirs.data_ptr(), P, C, L, flags, taps,
                                                   ctypes.c_void_p(stream), ctypes.byref(h)))
        else:
            _lib.check(self.lib.ss_bank_create_host(self.ctx, a.ctypes.data, P, C, L, flags, taps, ctypes.byref(h)))
        return RirBank(self, h, shape, normalize, taps, host, form)

    # ------------------------------------------------------------------ source pools
    def source_pool(self, candidates: T.Sequence[T.Union[MovingSource, StaticSource]],
                    levels: T.Optional[str] = None,
                    lufs_targets: T.Optional[T.Sequence[T.Optional[float]]] = None, sr: float = 16000) -> SourcePool:
        """Validate and upload a set of candidate sources once, for pooled slots (render.Pooled) of device plans to pick
        from at every run.  Every candidate is a MovingSource or StaticSource whose RIRs are a RirBank of this renderer
        (`dry`, `bounds`: contiguous CUDA tensors of its device; a moving candidate needs `bounds_host`), with no window,
        normalize_rirs or direct_taps (those belong to the slot and the bank); all share one kind (moving or static) and
        C, and may differ in L (e.g. the speakers of one formats.load_rir_dump, each with its own length): a slot that
        picks a candidate renders it with that candidate's own RIR partitions.  The pool's L, which its slots are given,
        is the longest candidate's.  The candidates' tensors and banks are kept alive by the pool.

        Candidates whose banks are all host banks (rir_bank(..., host=True)) make a host pool (`resident` "host"): its
        dry signals are copied into pinned host memory at once, so `dry` (and `bounds`, when `bounds_host` is not given)
        may also be NumPy arrays or CPU tensors; every plan run then copies only the rows and samples its slots read to
        the device (one more kernel launch per run).  A pool that mixes host and device banks is refused.  Over tap-form
        host banks (rir_bank(..., form="taps")) each run copies the staged rows' taps and transforms them on the device
        (one more launch again), with the bits of the same pool over spectral host banks; a pool that mixes forms is
        refused.

        `levels` = "mono" or "channels" also builds every candidate's level table (ss_pool_levels: the float64 prefix
        sums of the squares of its whole rendered stem, channel-folded like Mixture(mono=True) for "mono"), which
        CropDraw reads to test crops for silence; 8 bytes per sample.  The call then returns when the tables are
        complete.  They describe the dry signals as they are now: new signals need a new pool.

        `lufs_targets` (one float per candidate, or None to leave that candidate unscaled) loudness-normalises every
        candidate's whole stem as SonicSet stored it (get_lufs_norm_audio, SonicSet.py:97-101; `sr` the sample rate):
        each candidate is rendered whole once, measured like render_host(..., lufs_targets=) measures it, and every
        pooled slot that picks it stores its crops, direct stem included, times that (float32) gain.  The level tables
        then describe the normalised stems.  `loudness` holds the measured (LUFS, gain) pairs."""
        import torch
        if levels not in LEVELS:
            raise ValueError("source_pool: levels must be None, 'mono' or 'channels', got %r" % (levels,))
        n = len(candidates)
        if not 1 <= n <= 1 << 24:
            raise ValueError("source_pool: a pool holds 1 to 2^24 candidates, got %d" % n)
        _check_lufs("source_pool", "candidate", lufs_targets, n, sr)
        items = (SsSource * n)()
        keep = []
        first, L_max, host, form, sizes = None, 0, None, None, []
        for i, s in enumerate(candidates):
            if not isinstance(s, (MovingSource, StaticSource)):
                raise ValueError("source_pool: candidate %d must be a MovingSource or StaticSource, got %s"
                                 % (i, type(s).__name__))
            rb, _, P, C, L, mode = _rirs(s)
            if rb is None:
                raise ValueError("source_pool: candidate %d must take its RIRs from a RirBank" % i)
            _check_usable(rb, self, "source_pool: the RirBank of candidate %d" % i)
            if s.window is not None or s.normalize_rirs or int(s.direct_taps):
                raise ValueError("source_pool: candidate %d has a window, normalize_rirs or direct_taps; those belong to "
                                 "the pooled slot (render.Pooled) and the bank" % i)
            kind = (mode, C)
            if first is None:
                first = kind
            elif kind != first:
                raise ValueError("source_pool: candidate %d is (%s, C=%d), candidate 0 (%s, C=%d): every candidate has "
                                 "one kind and C (L may differ)" % ((i,) + _kind(kind) + _kind(first)))
            if host is None:
                host = rb.host
            elif rb.host != host:
                raise ValueError("source_pool: candidate %d has a %s bank, candidate 0 a %s one: a pool's banks are all "
                                 "host banks or all device banks" % ((i,) + (("host", "device") if rb.host else
                                                                           ("device", "host"))))
            if form is None:
                form = rb.form
            elif rb.form != form:
                raise ValueError("source_pool: candidate %d has a bank of form %r, candidate 0 one of form %r: a pool's "
                                 "banks are all of one form" % (i, rb.form, form))
            L_max = max(L_max, L)
            own = "candidate %d" % i
            bounds_host = s.bounds_host if mode == _lib.SS_MOVING_BOUNDS else None
            if host:                                       # copied into the pool: NumPy, CPU or CUDA tensors
                x, N = _pool_host_dry(s.dry, "source_pool", own, self.device, keep)
                if mode == _lib.SS_MOVING_BOUNDS and bounds_host is None and s.bounds is not None and \
                        not (_is_tensor(s.bounds) and s.bounds.is_cuda):
                    bounds_host = s.bounds.numpy() if _is_tensor(s.bounds) else s.bounds
            else:
                x = _tensor(s.dry, "source_pool", own, "dry", torch.float32, self.device)
                N = s.dry.numel()
            sizes.append(N)
            items[i] = SsSource(x=x, N=N, P=P, C=C, L=L, mode=mode, rir_bank=rb._h.value)
            if mode == _lib.SS_MOVING_BOUNDS:
                if not host:
                    items[i].bounds = _tensor(s.bounds, "source_pool", own, "bounds", torch.int32, self.device, (P,))
                if bounds_host is None:
                    raise ValueError("source_pool: moving candidate %d needs bounds_host" % i)
                bh = _bounds(bounds_host, P, "source_pool: bounds_host of %s" % own, keep)
                items[i].bounds_host = bh.ctypes.data
        if lufs_targets is not None and first[1] > 8:
            raise ValueError("source_pool: loudness normalisation supports at most 8 channels, the candidates have %d"
                             % first[1])
        loud = np.full((n, 2), np.nan, dtype=np.float64)
        post = _post_lufs(lufs_targets, items, sr, loud, keep)
        h = ctypes.c_void_p()
        _lib.check(self.lib.ss_pool_create(self.ctx, items, n, ctypes.byref(h)))
        st = self.lib.ss_pool_loudness(h, post) if post is not None else _lib.SS_OK
        if st == _lib.SS_OK and levels is not None:
            st = self.lib.ss_pool_levels(h, LEVELS[levels])        # tables of the normalised stems
        if st != _lib.SS_OK:
            self.lib.ss_pool_destroy(h)
            _lib.check(st)
        taps = {_rirs(s)[0].direct_taps for s in candidates}
        return SourcePool(self, h, candidates, first[0], first[1], L_max, min(sizes),
                          taps.pop() if len(taps) == 1 else 0, levels, loud, sizes, "host" if host else "device",
                          post is not None)

    # ------------------------------------------------------------------ dry pools
    def dry_pool(self, signals: T.Sequence[T.Any], levels: bool = False, host: bool = False,
                 dtype: str = "float32") -> DryPool:
        """A DryPool over `signals`: 1 to 2^24 contiguous 1-D CUDA float32 tensors of this renderer's device, referenced
        (not copied) and kept alive by the pool, for dry-picked pooled slots (DryPick) of device plans.  `levels` also
        builds every signal's level table, which start draws (CropDraw) test dry-picked speakers with; the call then
        returns when the tables are complete, and they describe the signals as they are now.

        With `host` True the pool is host-resident (`resident` "host"): the signals, which may also be 1-D NumPy arrays
        or CPU tensors, are copied into pinned host memory at once and not held, the level tables stay there too, and
        every plan run copies only the samples its dry-picked slots' crops read to the device.  Slots of host source
        pools take dry picks only from a host or a 16-bit dry pool.

        With `dtype` "int16" the pool is 16-bit: every signal, an int16 NumPy array or CPU / CUDA tensor, or a float one
        whose every sample is exactly k / 32768 (-32768 <= k <= 32767; 16-bit PCM as torchaudio or soundfile load it),
        of 1 to 2^23 samples, is copied as its int16 samples into an arena the pool owns (device memory, or pinned host
        memory with `host`), and its level tables are kept at one entry per 64 samples.  The pool renders, draws and
        measures bit for bit as the float32 pool of the same values, and serves slots of host source pools too."""
        import torch
        n = len(signals)
        if not 1 <= n <= 1 << 24:
            raise ValueError("dry_pool: a dry pool holds 1 to 2^24 signals, got %d" % n)
        if dtype not in ("float32", "int16"):
            raise ValueError("dry_pool: dtype must be \"float32\" or \"int16\", got %r" % (dtype,))
        ptrs = (ctypes.c_void_p * n)()
        lengths = np.empty(n, np.int32)
        keep = []
        if dtype == "int16":
            for i, x in enumerate(signals):
                ptrs[i], lengths[i] = _as_i16(x, "signal %d" % i, self.device, keep)
            torch.cuda.current_stream(self.device).synchronize()   # copied on the library's own streams
            flags = (_lib.SS_DRY_LEVELS if levels else 0) | (_lib.SS_DRY_HOST if host else 0)
            h = ctypes.c_void_p()
            _lib.check(self.lib.ss_dry_pool_create_i16(self.ctx, ptrs, lengths.ctypes.data, n, flags, ctypes.byref(h)))
            return DryPool(self, h, [], lengths, levels, "host" if host else "device", "int16")
        for i, x in enumerate(signals):
            own = "signal %d" % i
            if host:                                       # copied into the pool: NumPy, CPU or CUDA tensors
                ptrs[i], N = _pool_host_dry(x, "dry_pool", own, self.device, keep)
            else:
                ptrs[i], N = _tensor(x, "dry_pool", own, "dry", torch.float32, self.device), x.numel()
            if _is_tensor(x) and x.is_cuda and (x.dim() != 1 or N < 1):
                raise ValueError("dry_pool: %s must be 1-D and not empty, got shape %s" % (own, tuple(x.shape)))
            if N > 0x7fffffff - 16384:
                raise ValueError("dry_pool: %s has %d samples, at most %d" % (own, N, 0x7fffffff - 16384))
            lengths[i] = N
        if levels or host:                     # tables and copies are made on the library's own streams: finish the writes
            torch.cuda.current_stream(self.device).synchronize()
        flags = (_lib.SS_DRY_LEVELS if levels else 0) | (_lib.SS_DRY_HOST if host else 0)
        h = ctypes.c_void_p()
        _lib.check(self.lib.ss_dry_pool_create(self.ctx, ptrs, lengths.ctypes.data, n, flags, ctypes.byref(h)))
        return DryPool(self, h, [] if host else signals, lengths, levels, "host" if host else "device")

    def pair_gains(self, pool: SourcePool, dry_pool: DryPool, lufs_targets, sr: float = 16000) -> PairGains:
        """Measure the whole-stem loudness of every (dry signal d, candidate i) pair of `pool` and `dry_pool` once, for
        dry-picked slots (DryPick(dry_pool, pick, gains=...)) to store their stems at SonicSet's loudness
        (get_lufs_norm_audio, SonicSet.py:97-101) with no work per run.  `lufs_targets`: one float for every pair, or an
        (n_dry, n) array whose entry [d, i] is pair (d, i)'s target, NaN to leave that pair at gain 1 - SonicSet's
        per-stem draw is np.random.uniform(-19, -15, (n_dry, n)).  Each measured pair is candidate i rendered whole with
        the first N samples of signal d, measured like render_host(..., lufs_targets=) measures it: `loudness` holds
        the (LUFS, gain) pairs, bit for bit what render_host reports for that pair.  The call returns when the table is
        on the device (4 bytes per pair)."""
        import torch
        if not isinstance(pool, SourcePool):
            raise ValueError("pair_gains: pool must be a SourcePool, got %s" % type(pool).__name__)
        if not isinstance(dry_pool, DryPool):
            raise ValueError("pair_gains: dry_pool must be a DryPool, got %s" % type(dry_pool).__name__)
        _check_usable(pool, self, "pair_gains: the SourcePool")
        _check_usable(dry_pool, self, "pair_gains: the DryPool")
        n, n_dry = pool.n, dry_pool.n
        if n * n_dry > 1 << 26:
            raise ValueError("pair_gains: %d x %d pairs, at most 2^26" % (n_dry, n))
        if pool.C > 8:
            raise ValueError("pair_gains: loudness normalisation supports at most 8 channels, the pool has %d" % pool.C)
        if dry_pool.n_min < max(pool._sizes):
            raise ValueError("pair_gains: the DryPool holds a signal of %d samples, shorter than the pool's longest "
                             "candidate (N = %d)" % (dry_pool.n_min, max(pool._sizes)))
        t = np.asarray(lufs_targets, dtype=np.float64)
        if t.ndim == 0:
            t = np.full((n_dry, n), float(t))
        if t.shape != (n_dry, n):
            raise ValueError("pair_gains: lufs_targets must be a float or an (n_dry, n) = (%d, %d) array, got shape %s"
                             % (n_dry, n, t.shape))
        bad = np.argwhere(np.isinf(t))
        if len(bad):
            d, i = (int(v) for v in bad[0])
            raise ValueError("pair_gains: the loudness target of pair (%d, %d) is not finite: %r" % (d, i, t[d, i]))
        if not float(sr) > 0:
            raise ValueError("pair_gains: sr must be > 0, got %r" % (sr,))
        t = np.ascontiguousarray(t)
        from .SonicSim_audio import gating_block_size, gating_plan
        post = (SsPostLufs * n)()
        plans = {}
        for i, N in enumerate(pool._sizes):
            if np.isnan(t[:, i]).all():
                continue                                   # no measured pair: no gating plan
            block = float(gating_block_size(N, sr))
            if N not in plans:
                plans[N] = gating_plan(N, float(sr), block)
            brk, blo, bhi = plans[N]
            post[i] = SsPostLufs(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data,
                                 n_e=len(brk) - 1, n_blocks=len(blo), rate=float(sr), block_size=block)
        loud = np.full((n_dry, n, 2), np.nan, dtype=np.float64)
        if dry_pool.resident == "device":                  # measured on the library's own stream: finish the writes
            torch.cuda.current_stream(self.device).synchronize()
        h = ctypes.c_void_p()
        _lib.check(self.lib.ss_pair_gains_create(self.ctx, pool._h, dry_pool._h, post, t.ctypes.data,
                                                 loud.ctypes.data, ctypes.byref(h)))
        return PairGains(self, h, pool, dry_pool, loud)

    # ------------------------------------------------------------------ host buffers
    def plan_host(self, sources: T.Sequence[T.Union[MovingSource, StaticSource]],
                  outs: T.Optional[T.Sequence[np.ndarray]] = None,
                  lufs_targets: T.Optional[T.Sequence[T.Optional[float]]] = None, sr: float = 16000,
                  direct_outs: T.Optional[T.Sequence[T.Optional[np.ndarray]]] = None) -> "HostPlan":
        """Validate a batch once and bind it to its host buffers; `plan.run()` then renders it with a single
        C-ABI call (a generation loop refills the same pinned buffers and calls run() again).
        See render_host for the arguments."""
        _refuse_pooled(sources, "plan_host")
        n = len(sources)
        direct_outs = _check_direct_outs(direct_outs, n)
        _check_lufs("plan_host", "source", lufs_targets, n, sr)
        items = (SsSource * n)()
        results_l = np.full((n, 2), np.nan, dtype=np.float64)
        keep = []
        results = []
        for i, s in enumerate(sources):
            x = _as_f32(s.dry).reshape(-1)
            rb, h, P, C, L, mode = _rirs(s, lambda a, *_: _as_f32(a))
            bounds = _bounds(s.bounds, P, "bounds of source %d" % i, keep) if mode == _lib.SS_MOVING_BOUNDS else None
            N = x.shape[0]
            ws, wl, n_out = _window(s, i, N)
            shape = "(C, N)" if s.window is None else "(C, length) of its window"
            out = outs[i] if outs is not None else np.empty((C, n_out), dtype=np.float32)
            if out.shape != (C, n_out) or out.dtype != np.float32 or not out.flags.c_contiguous:
                raise ValueError("out[%d] must be C-contiguous float32 of shape %s" % (i, shape))
            dout = direct_outs[i]
            flags = _flags(s, i, dout)
            if dout is not None and (not isinstance(dout, np.ndarray) or dout.shape != (C, n_out) or
                                     dout.dtype != np.float32 or not dout.flags.c_contiguous):
                raise ValueError("direct_outs[%d] must be C-contiguous float32 of shape %s" % (i, shape))
            items[i] = SsSource(x=x.ctypes.data, rir=h.ctypes.data if h is not None else None, out=out.ctypes.data,
                                bounds=bounds.ctypes.data if bounds is not None else None,
                                N=N, P=P, C=C, L=L, mode=mode, flags=flags,
                                out_direct=dout.ctypes.data if dout is not None else None,
                                direct_taps=int(s.direct_taps), win_start=ws, win_len=wl,
                                rir_bank=_bank_of(self, s, i, P, C, L) if rb is not None else None)
            keep.append((x, h, out, dout, rb))
            results.append(out)
            if lufs_targets is not None and lufs_targets[i] is not None:
                if s.window is not None:
                    raise ValueError("source %d has a window and a loudness target: the loudness of a stem is "
                                     "measured over the whole stem" % i)
                if C > 8:
                    raise ValueError("loudness normalisation supports at most 8 channels")
        post = _post_lufs(lufs_targets, items, sr, results_l, keep)
        return HostPlan(self, items, post, n, results, results_l, keep, sources)

    def render_host(self, sources: T.Sequence[T.Union[MovingSource, StaticSource]],
                    outs: T.Optional[T.Sequence[np.ndarray]] = None,
                    lufs_targets: T.Optional[T.Sequence[T.Optional[float]]] = None, sr: float = 16000,
                    loudness_out: T.Optional[list] = None,
                    direct_outs: T.Optional[T.Sequence[T.Optional[np.ndarray]]] = None) -> T.List[np.ndarray]:
        """Render every source; returns a list of (C, N) float32 arrays (pinned `outs` may be passed).
        `lufs_targets[i]` (or None) additionally normalises stem i to that integrated loudness on
        the device before the copy out - SonicSim_audio.lufs_norm fused behind the render
        (SonicSet.py:97-101).  `loudness_out`, if a list, receives (measured LUFS, linear gain) per source.
        `direct_outs[i]`: a (C, N) float32 array that receives the direct-path stem of a source with direct_taps > 0
        (None for the other sources); with a loudness target it is scaled by the reverberant stem's gain.
        A source with a `window` (start, length) renders (C, length) arrays instead - the samples
        [start, start + length) of its full render, bit for bit - and reads and copies only what those need; it
        cannot have a loudness target."""
        plan = self.plan_host(sources, outs, lufs_targets, sr, direct_outs)
        res = plan.run()
        if loudness_out is not None and lufs_targets is not None:
            loudness_out[:] = plan.loudness()
        return res

    # ------------------------------------------------------------------ device tensors
    def render_device(self, sources, outs, stream: T.Optional[int] = None, direct_outs=None):
        """`sources`: MovingSource / StaticSource whose fields are CUDA float32 / int32 tensors;
        `outs`: preallocated CUDA (C, N) tensors - (C, length) for a source with a `window`; `direct_outs`: the same
        for the direct-path stems of sources with direct_taps > 0, None for the others.  Asynchronous on `stream`
        (default: torch's current stream of this renderer's device).  A window's start may be a CUDA int32 tensor (see MovingSource.window); a crop that
        moves every step is cheaper through a plan_device whose start tensors are rewritten between runs."""
        _refuse_pooled(sources, "render_device")
        items, n, keep = self._device_items(sources, outs, direct_outs)
        if stream is None:
            import torch
            stream = torch.cuda.current_stream(self.device).cuda_stream
        _lib.check(self.lib.ss_render_dev(self.ctx, items, n, ctypes.c_void_p(stream)))

    def plan_device(self, sources, outs, direct_outs=None, mixtures=None, draws=None, layouts=None,
                    values=None) -> "DevicePlan":
        """Bind a batch of device-resident sources to its output tensors once; `plan.run()` then renders it with a
        single C-ABI call - one CUDA graph launch (ss_plan_run; a generation loop overwrites the same tensors and
        calls run() again).  Every tensor must be a contiguous CUDA tensor of this renderer's device: float32 dry
        (N,), RIRs (P, C, L) / (C, L), outs[i] (C, N) for that source's own C and N ((C, length) with a `window`);
        int32 bounds (P,); direct_outs[i] as outs[i] for a source with direct_taps > 0, else None.  The plan binds
        each window's length, and its start when that is an int.  A start given as a one-element CUDA int32 tensor
        (e.g. starts[k] of a (B,) tensor; stems of one scene may share one element) is read on the device at every
        run: write new starts on the run's stream (starts.copy_(...)) and call run() again - crops that move every
        step, with no host work beyond the graph launch.  Such a plan transforms every RIR row of a raw-RIR source at
        every run; pass a RirBank to transform them once.

        `mixtures`: Mixture entries over the plan's stems, assembled at every run after the renders, inside the same
        graph launch (4 more kernel launches per run).  A training step of the separation dataloader is then

            starts.copy_(torch.randint(...)); sirs.uniform_(-6, 6); snr.uniform_(10, 20)   # movingdatamodule.py:106, :119
            plan.run()                                          # crops, gains and mixtures of every scene

        and the model takes (mix, speakers_out) from there; rms_db (Mixture) carries each speaker's level.  A Mixture
        with `direct_out` also writes its speakers' dereverberation targets in the same launches (ss_plan_create_target):
        the model then takes (mix, direct_out) for separation + dereverberation.

        `draws`: CropDraw entries, the dataloader's silence rule on the device: at the head of every run (one more
        kernel launch), each draw picks its readers' start from its `u`, rejecting starts at which a speaker's crop is
        below the threshold, before anything reads that start.  A step is then

            u.uniform_(); picks.copy_(...); sirs.uniform_(-6, 6); snr.uniform_(10, 20)
            plan.run()

        A Pooled slot with `dry` = DryPick(dry_pool, pick) also takes its dry signal from a DryPool at every run, so
        that every (dry signal, trajectory) pair is reachable in the same single graph launch
        (dry_picks.random_(0, n) before the run).  With `dry` = DryStream(utterance_pool, ids, offsets) the slot's dry
        stream is laid out from a 16-bit utterance pool at every run (ss_plan_create_stream): a fresh arrangement of
        utterances and gaps per step (dry.long_audio_layouts into the ids and offsets before the run).  With `dry` =
        BackgroundStream(clip_pool, ids, offsets, heads, counts) the slot's noise or music bed is laid out from a clip
        pool at every run (ss_plan_create_bg; dry.background_audio_layouts into the four arrays before the run).

        `layouts`: LayoutDraw entries, stream and bed slots whose layouts the plan draws itself at the head of every run
        (ss_plan_create_layout, one kernel launch more per run) instead of the caller's refresh.

        `values`: ValueDraw entries, the per-run values (picks, dry picks, starts, sirs, snr, a CropDraw's u, StemLoudness
        targets) that the plan draws itself at the head of every run (ss_plan_create_values, one kernel launch more per
        run).  With scene-major speaker pools (3 candidates per scene) and per-scene noise pools, the separation step
        (movingdatamodule.py:56-126) is

            values = [ValueDraw(scene, rng, 0, SCENES),                 # random.choice; noise slots pick scene[b]
                      ValueDraw(picks, rng, 0, 3, distinct=True, base=scene, stride=3),   # random.sample(range(1, 4), S)
                      ValueDraw(sirs, rng, -6, 6), ValueDraw(snr, rng, 10, 20),
                      ValueDraw(u, rng)]                                # CropDraw variates, (B, 101) float64
            plan = R.plan_device(srcs, outs, mixtures=mixes, draws=draws, layouts=layouts, values=values)
            ...
            rng[1] += 1                                                 # the whole step's randomness
            plan.run()

        Plain starts (`ValueDraw(starts, rng, 0, N - length + 1)`), dry picks and loudness targets (float64, e.g.
        U(-19, -15) for speech, U(-26, -22) for noise and U(-31, -27) for music, one tensor per range) are drawn the same
        way.

        With stream slots over a 16-bit pool in speaker order (paths, bounds = dry.speaker_groups(speaker_dirs), G =
        len(bounds) - 1), the step also draws each example's S distinct speakers (SonicSet.py:198) and lays every stream
        out from its speaker's utterances alone (create_long_audio over one speaker directory), in the same launches
        (ss_plan_create_groups):

            values = [ValueDraw(spk, rng, 0, G, distinct=True), ...]    # np.random.choice(speech_list, S, False)
            layouts = [LayoutDraw(slot_of[b][k], rng, 60 * 16000, groups=bounds, group=spk[b, k:k + 1])
                       for b in range(B) for k in range(S)]"""
        dry = self._device_dry(sources)
        streams = self._device_streams(sources)
        bgs = self._device_bgs(sources)
        items, n, keep = self._device_items(sources, outs, direct_outs)
        targets = []
        mixes = self._device_mixes(mixtures, outs, keep, items, targets) if mixtures else None
        drw = self._device_draws(draws, sources, keep) if draws else None
        lufs = self._device_lufs(sources, (outs, direct_outs, mixtures, draws), keep)
        grouped = []
        lay = self._device_layouts(layouts, sources, (outs, direct_outs, mixtures, draws), keep, grouped) \
            if layouts else None
        grp = (_lib.SsLayoutGroup * len(grouped))(*grouped) if grouped else None
        val = self._device_values(values, sources, (outs, direct_outs, mixtures, draws, layouts), keep) \
            if values else None
        trj = self._device_trajectories(sources, draws, (outs, direct_outs, mixtures, draws, layouts, values))
        return DevicePlan(self, items, n, keep, mixes, drw, dry, self._device_pair_gains(sources) if dry else None,
                          (_lib.SsPlanTarget * len(targets))(*targets) if targets else None, streams, bgs, lufs, lay,
                          val, grp, trj)

    def _device_trajectories(self, sources, draws, others):
        """Validated ss_trajectory array of a plan's slots with a Trajectory, or None without any.  `others`: the plan's
        other arguments, whose tensors no path or bounds may meet."""
        import torch
        entries, held = [], []
        speakers = {int(k) for d in (draws or ()) if isinstance(d, CropDraw) for k in d.speakers}
        for i, s in enumerate(sources):
            t = getattr(s, "trajectory", None)
            if t is None:
                continue
            if not isinstance(t, Trajectory):
                raise ValueError("plan_device: the trajectory of source %d must be a Trajectory" % i)
            pl = s.pool
            if pl.mode != _lib.SS_MOVING_BOUNDS:
                raise ValueError("plan_device: source %d has a Trajectory over a static pool" % i)
            if pl.resident != "device":
                raise ValueError("plan_device: source %d has a Trajectory over a host pool, whose staging is sized from "
                                 "its candidates' own bounds" % i)
            if pl.gains:
                raise ValueError("plan_device: source %d has a Trajectory over a pool with loudness gains, which were "
                                 "measured with the candidates' own timing" % i)
            d = s.dry
            if isinstance(d, DryPick) and d.gains is not None:
                raise ValueError("plan_device: source %d has a Trajectory and a DryPick with pair gains, which were "
                                 "measured with the candidates' own timing" % i)
            if i in speakers and not isinstance(d, (DryPick, DryStream)):
                raise ValueError("plan_device: source %d has a Trajectory and is a CropDraw speaker that renders its "
                                 "candidate's own dry signal, whose level table describes the stored timing" % i)
            own = "source %d" % i
            path = _tensor(t.path, "plan_device", own, "trajectory path", torch.int32, self.device, count=(3, 3))
            bounds = _tensor(t.bounds, "plan_device", own, "trajectory bounds", torch.int32, self.device,
                             (pl.p_max,))
            entries.append(_lib.SsTrajectory(slot=i, path_dev=path, bounds_dev=bounds))
            held.append(t)
        if not entries:
            return None
        # a path or bounds meets no other tensor the plan reads or writes, nor another path or bounds.  Trajectories
        # are attributes outside the Pooled tuples, so no span below is a path or bounds as such: a tensor met here is
        # one the plan also uses for something else, whatever object holds it.
        pools = [s.pool for s in sources if isinstance(s, Pooled)]
        tensors = _cuda_tensors((sources, others, [tuple(p.candidates) for p in pools]))
        spans = [(x.data_ptr(), x.data_ptr() + x.numel() * x.element_size()) for x in tensors]
        seen = []
        for e, t in zip(entries, held):
            for x in (t.path, t.bounds):
                lo, hi = x.data_ptr(), x.data_ptr() + x.numel() * x.element_size()
                if any(a < hi and lo < b for a, b in spans) or any(a < hi and lo < b for a, b in seen):
                    raise ValueError("plan_device: the trajectory of source %d meets another tensor of the plan"
                                     % e.slot)
                seen.append((lo, hi))
        return (_lib.SsTrajectory * len(entries))(*entries)

    def _device_dry(self, sources):
        """Validated ss_dry_pick array of a plan's dry-picked slots, or None without any."""
        import torch
        picks = []
        for i, s in enumerate(sources):
            d = getattr(s, "dry", None)
            if not isinstance(s, Pooled):
                if isinstance(d, DryPick):
                    raise ValueError("plan_device: source %d has a DryPick but is not a pooled slot (render.Pooled)" % i)
                continue
            if d is None or isinstance(d, (DryStream, BackgroundStream)):
                continue
            if not isinstance(d, DryPick):
                raise ValueError("plan_device: the dry of pooled source %d must be a DryPick or None, or a DryStream or a "
                                 "BackgroundStream" % i)
            if not isinstance(d.pool, DryPool):
                raise ValueError("plan_device: the dry pool of source %d must be a DryPool" % i)
            _check_usable(d.pool, self, "plan_device: the DryPool of source %d" % i)
            pl = s.pool
            if isinstance(pl, SourcePool):
                if pl.resident == "host" and d.pool.resident == "device" and d.pool.dtype == "float32":
                    raise ValueError("plan_device: pooled source %d has a dry pick over a host pool, whose runs stage "
                                     "each candidate's own dry signal" % i)
                if pl.gains and d.gains is None:
                    raise ValueError("plan_device: pooled source %d has a dry pick over a pool with loudness gains, "
                                     "which were measured with the candidates' own dry signals; give the DryPick "
                                     "pair gains (Renderer.pair_gains)" % i)
                if d.pool.n_min < max(pl._sizes):
                    raise ValueError("plan_device: the DryPool of source %d holds a signal of %d samples, shorter than "
                                     "its pool's longest candidate (N = %d)" % (i, d.pool.n_min, max(pl._sizes)))
            if d.gains is not None:
                g = d.gains
                if not isinstance(g, PairGains):
                    raise ValueError("plan_device: the gains of the DryPick of source %d must be a PairGains" % i)
                _check_usable(g, self, "plan_device: the PairGains of source %d" % i)
                if g.pool is not pl or g.dry_pool is not d.pool:
                    raise ValueError("plan_device: the PairGains of source %d were measured over another SourcePool "
                                     "or DryPool than the slot's pool and its DryPick's" % i)
            pick = _tensor(d.pick, "plan_device", "source %d" % i, "dry pick", torch.int32, self.device, count=(1, 1))
            picks.append(_lib.SsDryPick(slot=i, pool=d.pool._h.value, pick_dev=pick))
        return (_lib.SsDryPick * len(picks))(*picks) if picks else None

    def _device_streams(self, sources):
        """Validated ss_dry_stream array of a plan's stream slots, or None without any."""
        import torch
        streams = []
        for i, s in enumerate(sources):
            d = getattr(s, "dry", None)
            if not isinstance(d, DryStream):
                continue
            if not isinstance(s, Pooled):
                raise ValueError("plan_device: source %d has a DryStream but is not a pooled slot (render.Pooled)" % i)
            if not isinstance(d.pool, DryPool):
                raise ValueError("plan_device: the utterance pool of source %d must be a DryPool" % i)
            _check_usable(d.pool, self, "plan_device: the DryPool of source %d" % i)
            if d.pool.dtype != "int16":
                raise ValueError("plan_device: the DryStream of source %d needs a 16-bit DryPool (dry_pool(..., "
                                 "dtype=\"int16\")): a float32 pool's crop energies are not exact" % i)
            pl = s.pool
            if isinstance(pl, SourcePool):
                if pl.gains:
                    raise ValueError("plan_device: pooled source %d has a DryStream over a pool with loudness gains: a "
                                     "stream has no fixed (dry signal, trajectory) pair to measure" % i)
                if max(pl._sizes) > 1 << 23:
                    raise ValueError("plan_device: pooled source %d has a DryStream over a pool whose longest "
                                     "candidate (N = %d) exceeds 2^23 samples" % (i, max(pl._sizes)))
            own = "source %d" % i
            m = d.ids.numel() if isinstance(d.ids, torch.Tensor) else 0
            ids = _tensor(d.ids, "plan_device", own, "stream ids", torch.int32, self.device, ("m",), (1, 128))
            off = _tensor(d.offsets, "plan_device", own, "stream offsets", torch.int32, self.device, (m,))
            streams.append(_lib.SsDryStream(slot=i, pool=d.pool._h.value, ids_dev=ids, offsets_dev=off, m=m))
        return (_lib.SsDryStream * len(streams))(*streams) if streams else None

    def _device_bgs(self, sources):
        """Validated ss_bg_stream array of a plan's bed slots, or None without any."""
        import torch
        bgs = []
        for i, s in enumerate(sources):
            d = getattr(s, "dry", None)
            if not isinstance(d, BackgroundStream):
                continue
            if not isinstance(s, Pooled):
                raise ValueError("plan_device: source %d has a BackgroundStream but is not a pooled slot "
                                 "(render.Pooled)" % i)
            if not isinstance(d.pool, DryPool):
                raise ValueError("plan_device: the clip pool of source %d must be a DryPool" % i)
            _check_usable(d.pool, self, "plan_device: the DryPool of source %d" % i)
            if isinstance(s.pool, SourcePool) and s.pool.gains:
                raise ValueError("plan_device: pooled source %d has a BackgroundStream over a pool with loudness gains: "
                                 "a bed has no fixed (dry signal, trajectory) pair to measure" % i)
            own = "source %d" % i
            m = d.ids.numel() if isinstance(d.ids, torch.Tensor) else 0
            ids = _tensor(d.ids, "plan_device", own, "bed ids", torch.int32, self.device, ("m",), (1, 128))
            ptr = [_tensor(a, "plan_device", own, "bed " + f, torch.int32, self.device, (m,))
                   for a, f in ((d.offsets, "offsets"), (d.heads, "heads"), (d.counts, "counts"))]
            bgs.append(_lib.SsBgStream(slot=i, pool=d.pool._h.value, ids_dev=ids, offsets_dev=ptr[0], heads_dev=ptr[1],
                                       counts_dev=ptr[2], m=m))
        return (_lib.SsBgStream * len(bgs))(*bgs) if bgs else None

    def _device_lufs(self, sources, others, keep):
        """Validated ss_stream_lufs array of a plan's loudness slots (StemLoudness of a DryStream or BackgroundStream),
        or None without any; the gating plans are appended to `keep`.  `others`: the plan's other arguments, whose
        tensors no result may meet."""
        import torch
        from .SonicSim_audio import gating_block_size, gating_plan
        entries, held, rates = [], [], set()
        for i, s in enumerate(sources):
            d = getattr(s, "dry", None)
            q = getattr(d, "lufs", None) if isinstance(d, (DryStream, BackgroundStream)) else None
            if q is None:
                continue
            if not isinstance(q, StemLoudness):
                raise ValueError("plan_device: the lufs of source %d must be a StemLoudness" % i)
            pl = s.pool
            if pl.resident != "device":
                raise ValueError("plan_device: source %d has a loudness target over a host pool: its whole stem would "
                                 "stage every bank row over PCIe at every run" % i)
            if len(set(pl._sizes)) > 1:
                raise ValueError("plan_device: source %d has a loudness target over a pool whose candidates differ in N "
                                 "(%d to %d samples)" % (i, min(pl._sizes), max(pl._sizes)))
            if pl.C > 8:
                raise ValueError("plan_device: loudness normalisation supports at most 8 channels, the pool of source %d "
                                 "has %d" % (i, pl.C))
            own = "source %d" % i
            target = _tensor(q.target, "plan_device", own, "loudness target", torch.float64, self.device, count=(1, 1))
            result = (_tensor(q.result, "plan_device", own, "loudness result", torch.float64, self.device, count=(2, 2))
                      if q.result is not None else None)
            sr = float(q.sr)
            if not sr > 0 or not math.isfinite(sr):
                raise ValueError("plan_device: the sr of the loudness target of source %d must be > 0, got %r" % (i, q.sr))
            rates.add(sr)
            if len(rates) > 1:
                raise ValueError("plan_device: the loudness targets of a plan must share one sr, got %s" % sorted(rates))
            N = pl._sizes[0]
            block = float(gating_block_size(N, sr))
            brk, blo, bhi = gating_plan(N, sr, block)
            keep.append((brk, blo, bhi))
            gating = SsPostLufs(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data, n_e=len(brk) - 1,
                                n_blocks=len(blo), rate=sr, block_size=block)
            entries.append(_lib.SsStreamLufs(slot=i, gating=gating, target_dev=target, result_dev=result))
            held.append(q)
        if not entries:
            return None
        # a result is written at every run: it meets no other tensor the plan reads or writes, nor another result
        tensors = {id(t): t for t in _cuda_tensors((sources, others, held))}
        spans = [(k, t.data_ptr(), t.data_ptr() + t.numel() * t.element_size()) for k, t in tensors.items()]
        seen = []
        for e, q in zip(entries, held):
            if q.result is None:
                continue
            lo, hi = e.result_dev, e.result_dev + 16
            if any(k != id(q.result) and a < hi and lo < b for k, a, b in spans) or any(a < hi and lo < b
                                                                                      for a, b in seen):
                raise ValueError("plan_device: the loudness result of source %d meets another tensor of the plan"
                                 % e.slot)
            seen.append((lo, hi))
        return (_lib.SsStreamLufs * len(entries))(*entries)

    def _device_layouts(self, layouts, sources, others, keep, grouped=None):
        """Validated ss_layout_draw array of a plan's layout draws; their select_lengths and group bounds arrays are
        appended to `keep`, and the ss_layout_group entry of each grouped draw to `grouped` (a list; None: the plan may
        have no grouped draw).  `others`: the plan's other arguments, whose tensors the drawn layouts may not meet."""
        import torch
        from . import dry as _dry
        arr = (_lib.SsLayoutDraw * len(layouts))()
        drawn, rngs, gtens = [], [], []                 # gtens: the group tensors of grouped draws
        for k, d in enumerate(layouts):
            if not isinstance(d, LayoutDraw):
                raise ValueError("plan_device: layout %d must be a LayoutDraw" % k)
            i = int(d.slot)
            s = sources[i] if 0 <= i < len(sources) else None
            w = getattr(s, "dry", None)
            if not isinstance(s, Pooled) or not isinstance(w, (DryStream, BackgroundStream)):
                raise ValueError("plan_device: layout %d names source %d, which is not a stream or bed slot (a Pooled "
                                 "slot with a DryStream or BackgroundStream)" % (k, i))
            if any(int(e.slot) == i for e in layouts[:k]):
                raise ValueError("plan_device: layout %d names source %d, which another layout draw names" % (k, i))
            own = "layout %d" % k
            bed = isinstance(w, BackgroundStream)
            bounds = None
            if d.groups is not None or d.group is not None:     # speaker groups: a stream slot's, both given
                if bed:
                    raise ValueError("plan_device: layout %d has speaker groups, but source %d is a bed slot: beds draw "
                                     "from the whole clip pool" % (k, i))
                if d.groups is None or d.group is None:
                    raise ValueError("plan_device: layout %d needs both groups and group, or neither" % k)
                bounds = np.ascontiguousarray(_dry._group_bounds(d.groups, w.pool.n, "plan_device: " + own),
                                              dtype=np.int32)
                gp = _tensor(d.group, "plan_device", own, "group", torch.int32, self.device, count=(1, 1))
                if grouped is None:
                    raise ValueError("plan_device: layout %d has speaker groups, which this call does not take" % k)
                keep.append(bounds)
                grouped.append(_lib.SsLayoutGroup(layout=k, n_groups=bounds.size - 1, bounds=bounds.ctypes.data,
                                                  group_dev=gp))
                gtens.append(d.group)
            rng = _tensor(d.rng, "plan_device", own, "rng", torch.int64, self.device, count=(2, 2))
            if rng % 8:
                raise ValueError("plan_device: the rng of layout %d must be 8-byte aligned" % k)
            total, sr = int(d.total), int(d.sample_rate)
            if not 1 <= total < 1 << 31 or not 1 <= sr <= 214748364:
                raise ValueError("plan_device: layout %d needs 1 <= total < 2^31 and 1 <= sample_rate <= 214748364 "
                                 "(10 s of samples in int32), got %d and %d" % (k, total, sr))
            sel = None
            if d.select_lengths is not None:
                if not bed:
                    raise ValueError("plan_device: layout %d has select_lengths, but source %d is a stream slot: only "
                                     "beds select by other lengths" % (k, i))
                sel = np.asarray(d.select_lengths.cpu() if _is_tensor(d.select_lengths) else d.select_lengths)
                if sel.shape != (w.pool.n,) or not np.issubdtype(sel.dtype, np.integer) or \
                        (sel.size and (sel.min() < 0 or sel.max() >= 1 << 31)):
                    raise ValueError("plan_device: the select_lengths of layout %d must be %d non-negative int32 "
                                     "lengths, one per clip" % (k, w.pool.n))
                sel = np.ascontiguousarray(sel, dtype=np.int32)
                keep.append(sel)
            K = (_dry.background_audio_max_selected(sel if sel is not None else w.pool.sizes, total) if bed
                 else _dry.long_audio_max_selected(w.pool.sizes, total, bounds))
            if K > 1024:
                raise ValueError("plan_device: layout %d could select %d %s, at most 1024%s" %
                                 (k, K, "clips" if bed else "utterances", " in one group" if bounds is not None else ""))
            arrays = (w.ids, w.offsets) + ((w.heads, w.counts) if bed else ())
            drawn += [a for a in arrays if _is_tensor(a)]
            rngs.append(d.rng)
            arr[k] = _lib.SsLayoutDraw(slot=i, rng_dev=rng, total=total, sample_rate=sr,
                                       select_lengths=sel.ctypes.data if sel is not None else None)
        # a drawn layout is written at every run: it meets no other tensor the plan reads or writes, another drawn
        # layout included; an rng meets nothing the plan writes
        outs, direct_outs, mixtures, draws = others
        stems = [getattr(s.dry, "lufs", None) for s in sources if isinstance(s, Pooled)]
        span = lambda t: (t.data_ptr(), t.data_ptr() + t.numel() * t.element_size())   # noqa: E731
        every = _cuda_tensors((sources, others, stems))
        for a in drawn:
            lo, hi = span(a)
            if sum(1 for t in every if t is a) + sum(1 for t in drawn if t is a) > 2 or \
                    any(t is not a and span(t)[0] < hi and lo < span(t)[1] for t in every):
                raise ValueError("plan_device: a layout tensor drawn by the plan meets another tensor of the plan")
        written = drawn + _cuda_tensors((outs, direct_outs, [q.result for q in stems if q is not None],
                                         [(m.mix, m.speakers_out, m.rms_db, m.direct_out) for m in mixtures or ()],
                                         [(d.start, d.used) for d in draws or ()]))
        for t in rngs:
            lo, hi = span(t)
            if any(a < hi and lo < b for a, b in map(span, written)):
                raise ValueError("plan_device: a layout draw's rng meets a tensor the plan writes")
        for t in gtens:                                # (a ValueDraw may write a group: _device_values checks that)
            lo, hi = span(t)
            if any(a < hi and lo < b for a, b in map(span, written)):
                raise ValueError("plan_device: a layout draw's group meets a tensor the plan writes")
        keep.append(list(layouts))
        return arr

    def _device_values(self, values, sources, others, keep):
        """Validated ss_value_draw array of a plan's value draws.  `others`: the plan's other arguments; a drawn `out`
        meets none of their tensors but the small per-run inputs it may write."""
        import torch
        kinds = {torch.float32: _lib.SS_VALUE_F32, torch.float64: _lib.SS_VALUE_F64, torch.int32: _lib.SS_VALUE_INT}
        if len(values) > 1 << 20:
            raise ValueError("plan_device: at most 2^20 value draws, got %d" % len(values))
        arr = (_lib.SsValueDraw * len(values))()
        span_of = []                                   # int32 draws: (least, most) value
        rows = None
        for r, v in enumerate(values):
            own = "value draw %d" % r
            if not isinstance(v, ValueDraw):
                raise ValueError("plan_device: %s must be a ValueDraw" % own)
            o = v.out
            if not _is_tensor(o) or o.dtype not in kinds:
                raise ValueError("plan_device: the out of %s must be a float32, float64 or int32 CUDA tensor" % own)
            _tensor(o, "plan_device", own, "out", o.dtype, self.device)
            if o.dim() not in (1, 2) or not 1 <= o.shape[0] <= 65535 or (o.dim() == 2 and not 1 <= o.shape[1] <= 4096):
                raise ValueError("plan_device: the out of %s must have shape (B,) or (B, k) with 1 <= B <= 65535 and "
                                 "1 <= k <= 4096, got %s" % (own, tuple(o.shape)))
            B, k = int(o.shape[0]), int(o.shape[1]) if o.dim() == 2 else 1
            if rows is not None and B != rows:
                raise ValueError("plan_device: %s has %d rows, value draw 0 has %d: every value draw of a plan has the "
                                 "same B" % (own, B, rows))
            rows = B
            rng = _tensor(v.rng, "plan_device", own, "rng", torch.int64, self.device, count=(2, 2))
            if rng % 8:
                raise ValueError("plan_device: the rng of %s must be 8-byte aligned" % own)
            kind = kinds[o.dtype]
            e = _lib.SsValueDraw(out=o.data_ptr(), rng_dev=rng, kind=kind, rows=B, k=k, base=-1)
            if kind != _lib.SS_VALUE_INT:
                low, high = float(v.low), float(v.high)
                if not (np.isfinite(low) and np.isfinite(high) and low < high):
                    raise ValueError("plan_device: %s needs finite low < high, got [%r, %r)" % (own, v.low, v.high))
                if kind == _lib.SS_VALUE_F32 and (float(np.float32(low)) != low or float(np.float32(high)) != high):
                    raise ValueError("plan_device: the bounds of float32 %s must be exact in float32, got [%r, %r)"
                                     % (own, low, high))
                if v.distinct or v.base is not None or v.stride:
                    raise ValueError("plan_device: distinct, base and stride are for int32 draws only (%s)" % own)
                e.low, e.high = low, high
                span_of.append(None)
            else:
                low, high = v.low, v.high
                if int(low) != low or int(high) != high or not -(1 << 31) <= int(low) < int(high) < 1 << 31:
                    raise ValueError("plan_device: int32 %s needs integer bounds -2^31 <= low < high < 2^31, got "
                                     "[%r, %r)" % (own, v.low, v.high))
                low, high = int(low), int(high)
                if v.distinct:
                    if k > 64 or k > high - low:
                        raise ValueError("plan_device: distinct %s samples k = %d of %d values, at most min(64, "
                                         "high - low)" % (own, k, high - low))
                    e.kind = _lib.SS_VALUE_DISTINCT
                e.ilow, e.ihigh = low, high
                lo, hi = low, high - 1
                if v.base is not None:
                    j = next((j for j in range(r) if values[j].out is v.base), None)
                    if j is None or span_of[j] is None or values[j].out.numel() != B:
                        raise ValueError("plan_device: the base of %s must be the (B,) out of an earlier int32 value "
                                         "draw" % own)
                    if int(v.stride) < 1:
                        raise ValueError("plan_device: %s needs stride >= 1 with a base, got %r" % (own, v.stride))
                    lo, hi = lo + span_of[j][0] * int(v.stride), hi + span_of[j][1] * int(v.stride)
                    if lo < -(1 << 31) or hi >= 1 << 31:
                        raise ValueError("plan_device: base * stride + value of %s may overflow int32" % own)
                    e.base, e.stride = j, int(v.stride)
                elif v.stride:
                    raise ValueError("plan_device: %s has a stride but no base" % own)
                span_of.append((lo, hi))
            arr[r] = e
        # an out meets nothing the plan reads or writes but the small per-run inputs; an rng meets nothing written
        outs, direct_outs, mixtures, draws, layouts = others
        starts = [d.start.data_ptr() for d in draws or () if _is_tensor(d.start)]
        lufs = [q for s in sources for q in [getattr(getattr(s, "dry", None), "lufs", None)] if q is not None]
        inputs = [q.target for q in lufs]
        stems = []                                     # (a DryStream's lufs lies outside its tuple)
        for s in sources:
            if not isinstance(s, Pooled):
                continue
            inputs.append(s.pick)
            if _is_tensor(s.window[0]) and s.window[0].data_ptr() not in starts:
                inputs.append(s.window[0])
            if isinstance(s.dry, DryPick):
                inputs.append(s.dry.pick)
            if isinstance(s.dry, DryStream) and s.dry.lufs is not None:
                stems.append(s.dry.lufs)
        inputs += [t for m in mixtures or () for t in (m.sirs, m.snr)] + [d.u for d in draws or ()]
        groups = [d.group for d in layouts or () if d.group is not None]      # (outside their LayoutDraw's tuple)
        inputs += groups                               # a grouped layout draw's group
        every = _cuda_tensors((sources, others, stems, groups))
        uses = collections.Counter(id(t) for t in every)
        uses.subtract(id(t) for t in inputs if _is_tensor(t))
        span = lambda t: (t.data_ptr(), t.data_ptr() + t.numel() * t.element_size())   # noqa: E731
        meets = lambda a, b: a[0] < b[1] and b[0] < a[1]                                  # noqa: E731
        other = [span(t) for t in every if uses[id(t)] > 0]
        drawn = [span(v.out) for v in values]
        rngs = [span(v.rng) for v in values]
        for r, a in enumerate(drawn):
            if any(meets(a, b) for b in other + rngs) or any(meets(a, b) for b in drawn[:r]):
                raise ValueError("plan_device: the out of value draw %d meets another tensor of the plan (only picks, "
                                 "dry picks, starts, sirs, snr, a CropDraw's u and StemLoudness targets may be drawn)" % r)
        written = [span(t) for t in _cuda_tensors((outs, direct_outs, [q.result for q in lufs],
                                                   [(m.mix, m.speakers_out, m.rms_db, m.direct_out)
                                                    for m in mixtures or ()],
                                                   [(d.start, d.used) for d in draws or ()]))]
        for d in layouts or ():
            w = sources[int(d.slot)].dry
            written += [span(t) for t in (w.ids, w.offsets) + ((w.heads, w.counts) if isinstance(w, BackgroundStream)
                                                               else ()) if _is_tensor(t)]
        for r, a in enumerate(rngs):
            if any(meets(a, b) for b in written):
                raise ValueError("plan_device: the rng of value draw %d meets a tensor the plan writes" % r)
        keep.append(list(values))
        return arr

    @staticmethod
    def _device_pair_gains(sources):
        """The ss_pair_gains handles of a plan's dry picks (the order of _device_dry), or None when no pick has gains."""
        picks = [s.dry for s in sources if isinstance(s, Pooled) and isinstance(s.dry, DryPick)]
        if all(d.gains is None for d in picks):
            return None
        return (ctypes.c_void_p * len(picks))(*[d.gains._h.value if d.gains is not None else None for d in picks])

    def _device_draws(self, draws, sources, keep):
        """Validated ss_plan_draw array of a plan's start draws; their tensors are appended to `keep`."""
        import torch
        n = len(sources)
        arr = (_lib.SsPlanDraw * len(draws))()
        seen = set()
        for k, d in enumerate(draws):
            own = "draw %d" % k
            start = _tensor(d.start, "plan_device", own, "start", torch.int32, self.device, count=(1, 1))
            u = _tensor(d.u, "plan_device", own, "u", torch.float64, self.device, count=(1, 4096))
            used = (_tensor(d.used, "plan_device", own, "used", torch.int32, self.device, count=(1, 1))
                    if d.used is not None else None)
            if start in seen:
                raise ValueError("plan_device: draw %d shares its start tensor with another draw" % k)
            seen.add(start)
            if used is not None and used == start:
                raise ValueError("plan_device: used of draw %d is its start tensor" % k)
            thr = float(d.threshold_db)
            if not np.isfinite(thr):
                raise ValueError("plan_device: threshold_db of draw %d must be finite, got %r" % (k, thr))
            spk = [int(v) for v in d.speakers]
            if not 1 <= len(spk) <= 8:
                raise ValueError("plan_device: draw %d must name 1 to 8 speakers, got %d" % (k, len(spk)))
            if len(set(spk)) != len(spk):
                raise ValueError("plan_device: draw %d names a speaker more than once" % k)
            readers = [i for i, s in enumerate(sources)
                       if s.window is not None and _is_tensor(s.window[0]) and s.window[0].data_ptr() == start]
            for i in readers:
                if not isinstance(sources[i], Pooled):
                    raise ValueError("plan_device: source %d reads the start of draw %d but is not a pooled slot "
                                     "(render.Pooled)" % (i, k))
            if len({int(sources[i].window[1]) for i in readers}) > 1:
                raise ValueError("plan_device: the readers of draw %d (sources %s) have different window lengths"
                                 % (k, readers))
            if len(readers) > 16:
                raise ValueError("plan_device: draw %d has %d readers, at most 16" % (k, len(readers)))
            for v in spk:
                if not 0 <= v < n:
                    raise ValueError("plan_device: draw %d names source %d of %d" % (k, v, n))
                if v not in readers:
                    raise ValueError("plan_device: speaker %d of draw %d does not take its window start from the "
                                     "draw's start tensor" % (v, k))
                dry = sources[v].dry
                if isinstance(dry, BackgroundStream):
                    raise ValueError("plan_device: speaker %d of draw %d is a bed slot (BackgroundStream): the draws "
                                     "test speakers only" % (v, k))
                if isinstance(dry, (DryPick, DryStream)):
                    if not dry.pool.levels:
                        raise ValueError("plan_device: speaker %d of draw %d: its DryPool has no level tables "
                                         "(dry_pool(levels=True))" % (v, k))
                elif sources[v].pool.levels is None:
                    raise ValueError("plan_device: speaker %d of draw %d: its SourcePool has no level tables "
                                     "(source_pool(levels=...))" % (v, k))
            e = arr[k]
            for i, v in enumerate(spk):
                e.speakers[i] = v
            e.start, e.u, e.used, e.S, e.tries, e.threshold_db = start, u, used, len(spk), d.u.numel(), thr
        keep.append(list(draws))
        return arr

    def _device_mixes(self, mixtures, outs, keep, items=None, targets=None):
        """Validated ss_plan_mix array of a plan's mixtures; their tensors are appended to `keep`.  A mixture with a
        direct_out needs `items` (the plan's SsSource array, whose speakers must render direct-path stems) and `targets`,
        a list that receives its validated SsPlanTarget."""
        import torch
        n = len(outs)
        arr = (_lib.SsPlanMix * len(mixtures))()
        for k, m in enumerate(mixtures):
            spk, noi = [int(v) for v in m.speakers], [int(v) for v in m.noises]
            S, M = len(spk), len(noi)
            if not 1 <= S <= 8 or not 1 <= M <= 8:
                raise ValueError("plan_device: mixture %d must have 1 to 8 speakers and 1 to 8 noises, got %d and %d"
                                 % (k, S, M))
            for v in spk + noi:
                if not 0 <= v < n:
                    raise ValueError("plan_device: mixture %d names source %d of %d" % (k, v, n))
            if len(set(spk + noi)) != S + M:
                raise ValueError("plan_device: mixture %d names a source more than once" % k)
            C, Tn = outs[spk[0]].shape
            for v in spk + noi:
                if tuple(outs[v].shape) != (C, Tn):
                    raise ValueError("plan_device: the stems of mixture %d must share one (C, T); source %d has %s, "
                                     "source %d has %s" % (k, spk[0], (C, Tn), v, tuple(outs[v].shape)))
            mono = bool(m.mono)
            row = (Tn,) if mono else (C, Tn)
            if S == 1 and m.sirs is not None:
                raise ValueError("plan_device: mixture %d has one speaker: its sirs must be None" % k)
            own, f32 = "mixture %d" % k, torch.float32
            sirs = (_tensor(m.sirs, "plan_device", own, "sirs", f32, self.device, count=(S - 1, S - 1))
                    if S > 1 else None)
            snr = _tensor(m.snr, "plan_device", own, "snr", f32, self.device, count=(1, 1))
            mix = _tensor(m.mix, "plan_device", own, "mix", f32, self.device, row)
            sp_out = (_tensor(m.speakers_out, "plan_device", own, "speakers_out", f32, self.device, (S,) + row)
                      if m.speakers_out is not None else None)
            rms = (_tensor(m.rms_db, "plan_device", own, "rms_db", f32, self.device, (S,))
                   if m.rms_db is not None else None)
            delay = int(m.noise_delay)
            if delay < 0:
                raise ValueError("plan_device: noise_delay of mixture %d must be >= 0, got %d" % (k, delay))
            if m.direct_out is not None:
                for v in spk:
                    if not items[v].out_direct:
                        raise ValueError("plan_device: mixture %d has a direct_out, but its speaker source %d renders no "
                                         "direct-path stem (direct_taps and a direct_outs entry)" % (k, v))
                d_out = _tensor(m.direct_out, "plan_device", own, "direct_out", f32, self.device, (S,) + row)
                targets.append(_lib.SsPlanTarget(mix=k, direct_out=d_out))
            e = arr[k]
            for i, v in enumerate(spk):
                e.speakers[i] = v
            for i, v in enumerate(noi):
                e.noises[i] = v
            e.S, e.M, e.sirs, e.snr, e.mix, e.speakers_out, e.rms_db = S, M, sirs, snr, mix, sp_out, rms
            e.flags, e.noise_delay = _lib.SS_MIX_MONO if mono else 0, delay
        keep.append(list(mixtures))
        return arr

    def _device_items(self, sources, outs, direct_outs=None):
        """Validated ss_source array of a device-resident batch: (items, n, objects to keep alive)."""
        import torch
        n = len(sources)
        if len(outs) != n:
            raise ValueError("plan_device: %d sources but %d output tensors" % (n, len(outs)))
        direct_outs = _check_direct_outs(direct_outs, n)
        items = (SsSource * n)()
        keep = [sources, outs, direct_outs]
        f32 = torch.float32
        for i, s in enumerate(sources):
            own = "source %d" % i
            if isinstance(s, Pooled):
                pl = s.pool
                if not isinstance(pl, SourcePool):
                    raise ValueError("plan_device: the pool of source %d must be a SourcePool" % i)
                _check_usable(pl, self, "plan_device: the SourcePool of source %d" % i)
                pick = _tensor(s.pick, "plan_device", own, "pick", torch.int32, self.device, count=(1, 1))
                if s.window is None:
                    raise ValueError("plan_device: pooled source %d needs a window (start, length)" % i)
                ws, wl, n_out, start = _window_dev(s, i, pl.n_min, self.device)
                taps = int(s.direct_taps)
                if taps > 0 and taps != pl.direct_taps:
                    raise ValueError("plan_device: pooled source %d has direct_taps = %d, but not every candidate's bank "
                                     "holds a direct set with these taps" % (i, taps))
                C = pl.C
                out = _tensor(outs[i], "plan_device", own, "out", f32, self.device, (C, n_out))
                items[i] = SsSource(out=out, C=C, L=pl.L, mode=pl.mode, pool=pl._h.value, pick_dev=pick)
            else:
                x = _tensor(s.dry, "plan_device", own, "dry", f32, self.device)
                N = s.dry.numel()
                ws, wl, n_out, start = _window_dev(s, i, N, self.device)

                def raw(t, field, shape):                  # raw RIRs: checked before _rirs reads their shape
                    _tensor(t, "plan_device", own, field, f32, self.device, shape)
                    return t
                rb, h, P, C, L, mode = _rirs(s, raw)
                out = _tensor(outs[i], "plan_device", own, "out", f32, self.device, (C, n_out))
                items[i] = SsSource(x=x, rir=h.data_ptr() if h is not None else None, out=out, N=N, P=P, C=C, L=L,
                                    mode=mode)
                if mode == _lib.SS_MOVING_BOUNDS:
                    items[i].bounds = _tensor(s.bounds, "plan_device", own, "bounds", torch.int32, self.device, (P,))
                    if s.bounds_host is not None:
                        items[i].bounds_host = _bounds(s.bounds_host, P, "plan_device: bounds_host of %s" % own,
                                                       keep).ctypes.data
                if rb is not None:
                    items[i].rir_bank = _bank_of(self, s, i, P, C, L)
            items[i].flags = _flags(s, i, direct_outs[i])
            items[i].win_start, items[i].win_len = ws, wl
            if start is not None:
                items[i].win_start_dev = start.data_ptr()         # kept alive with `sources`
            if direct_outs[i] is not None:
                items[i].out_direct = _tensor(direct_outs[i], "plan_device", own, "direct_out", f32, self.device,
                                              (C, n_out))
                items[i].direct_taps = int(s.direct_taps)
        return items, n, keep

    def check_device_errors(self):
        """Waits for the device and raises what the reference would have raised for a trajectory the device path met
        but could not refuse up front: IndexError for an interp_index outside [0, P - 2] (NumPy's fancy index at
        SonicSim_moving.py:89-90), ValueError for a device-side bounds table that is not ascending from 0 to N or for a
        window start tensor that held a value outside [0, N - length] (the window was rendered clamped into range);
        IndexError too for a pick, dry pick or grouped LayoutDraw's group outside its range (clamped into it), and
        ValueError for a Trajectory whose path or bounds were invalid at a run (the candidate's own path rendered)."""
        bits = ctypes.c_uint32()
        _lib.check(self.lib.ss_device_errors(self.ctx, ctypes.byref(bits)))
        if bits.value & 1:
            raise IndexError("an interp_index on the device was out of bounds for the number of RIR positions")
        if bits.value & 8:
            raise IndexError("a pick on the device was out of range for the candidates of its SourcePool; it was clamped "
                             "into [0, n)")
        if bits.value & 16:
            raise IndexError("a dry pick on the device was out of range for the signals of its DryPool; it was clamped "
                             "into [0, n)")
        if bits.value & 128:
            raise IndexError("a grouped LayoutDraw's group on the device was out of range for its G groups; it was "
                             "clamped into [0, G)")
        if bits.value & 2:
            raise ValueError("a device-side trajectory bounds table is not ascending from 0 to N")
        if bits.value & 4:
            raise ValueError("a window start on the device was outside [0, N - length]; the window was clamped into "
                             "that range")
        if bits.value & 32:
            raise ValueError("a DryStream or BackgroundStream layout on the device held an invalid entry (an id >= n, a "
                             "negative offset, a head and count outside the clip or an offset before the end of the "
                             "previous entry); it was skipped")
        if bits.value & 64:
            raise ValueError("a StemLoudness target on the device was not finite; that slot was stored unscaled")
        if bits.value & 256:
            raise ValueError("a Trajectory on the device held an invalid path or bounds table; that slot rendered its "
                             "candidate's own path")

    def launch_count(self) -> int:
        return int(self.lib.ss_launch_count(self.ctx))

    def reset_stats(self):
        self.lib.ss_reset_stats(self.ctx)

    def set_profiling(self, on: bool):
        _lib.check(self.lib.ss_set_profiling(self.ctx, 1 if on else 0))

    def get_profile(self):
        """(ms in k_spectra, ms in k_render, launch pairs) since the previous call."""
        a, b, n = ctypes.c_double(), ctypes.c_double(), ctypes.c_int64()
        _lib.check(self.lib.ss_get_profile(self.ctx, ctypes.byref(a), ctypes.byref(b), ctypes.byref(n)))
        return a.value, b.value, n.value

    def set_chunk_bytes(self, nbytes: int):
        _lib.check(self.lib.ss_set_chunk_bytes(self.ctx, int(nbytes)))


class DevicePlan:
    """A batch of device-resident sources bound to its output tensors (Renderer.plan_device): an ss_plan of the C ABI -
    descriptors, block tables and scratch resident on the device, the launches captured into a CUDA graph.  With
    mixtures, the plan also assembles them at every run; with draws, it first draws their starts; with dry picks, its
    dry-picked slots take their dry signals from dry pools, with pair gains their gains from pair-gain tables; with
    dereverberation targets its mixtures also write those, with stream slots it lays out their dry streams and with bed
    slots their noise and music beds, with loudness slots it measures their whole stems at every run, with layout draws
    it draws its stream and bed layouts at every run, with value draws it draws its per-run inputs at every run, with
    grouped layout draws it lays each such stream out from the group of utterances its group tensor names, with
    trajectories its slots follow the path and timing their Trajectory holds at every run.  Every plan is created by
    ss_plan_create_traj, with NULL and a count of 0 for each part it does not have."""

    def __init__(self, renderer, items, n, keep, mixes=None, draws=None, dry=None, pair_gains=None, targets=None,
                 streams=None, bgs=None, lufs=None, layouts=None, values=None, groups=None, trajectories=None):
        self.renderer, self.items, self.n, self._keep, self.mixes = renderer, items, n, keep, mixes
        self.draws, self.dry, self.pair_gains, self.targets, self.streams = draws, dry, pair_gains, targets, streams
        self.bgs, self.lufs, self.layouts, self.values, self.groups = bgs, lufs, layouts, values, groups
        self.trajectories = trajectories
        self._plan = ctypes.c_void_p()
        if n > 0:
            args = (renderer.ctx, items, n, mixes, len(mixes) if mixes else 0, draws, len(draws) if draws else 0, dry,
                    pair_gains, len(dry) if dry else 0, targets, len(targets) if targets else 0, streams,
                    len(streams) if streams else 0, bgs, len(bgs) if bgs else 0, lufs, len(lufs) if lufs else 0,
                    layouts, len(layouts) if layouts else 0, values, len(values) if values else 0, groups,
                    len(groups) if groups else 0, trajectories, len(trajectories) if trajectories else 0)
            _lib.check(renderer.lib.ss_plan_create_traj(*args, ctypes.byref(self._plan)))
        self._banks = _hold_banks(self, keep[0])

    def run(self, stream: T.Optional[int] = None):
        """Asynchronous on `stream` (default: torch's current stream of the renderer's device)."""
        if self.n == 0:
            return
        if stream is None:
            import torch
            stream = torch.cuda.current_stream(self.renderer.device).cuda_stream
        _lib.check(self.renderer.lib.ss_plan_run(self._plan, ctypes.c_void_p(stream)))

    def is_graph(self) -> bool:
        return self.n > 0 and self.renderer.lib.ss_plan_is_graph(self._plan) == 1

    def close(self):
        if self._plan:
            self.renderer.lib.ss_plan_destroy(self._plan)
            self._plan = ctypes.c_void_p()
        if getattr(self, "_banks", None) is not None:
            self._banks()                      # the plan no longer reads its banks: a closed one may be freed now

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class HostPlan:
    """A validated batch bound to its host input / output buffers (Renderer.plan_host)."""

    def __init__(self, renderer, items, post, n, results, results_l, keep, sources=()):
        self.renderer, self.items, self.post, self.n = renderer, items, post, n
        self.results, self.results_l, self._keep = results, results_l, keep
        self._banks = _hold_banks(self, sources)

    def run(self) -> T.List[np.ndarray]:
        """H2D -> render [-> loudness] -> D2H of the whole batch; returns the (C, N) output arrays."""
        _lib.check(self.renderer.lib.ss_render_host_ex(self.renderer.ctx, self.items, self.n, self.post))
        return self.results

    def loudness(self) -> T.List[T.Tuple[float, float]]:
        """(measured LUFS, linear gain) per source of the last run (NaN where no target was given)."""
        return [tuple(r) for r in self.results_l]


_default: T.Optional[Renderer] = None


def default_renderer() -> Renderer:
    global _default
    if _default is None:
        _default = Renderer()
    return _default


def trajectory_bounds(receiver_position, total_samples: int) -> np.ndarray:
    """Positions (P, 3) -> int32 segment bounds (P,), via the reference's constant-speed rule
    (SonicSim_moving.py:32-39; consumes the global NumPy RNG like the reference)."""
    return bounds_from_counts(_samples_per_interval(np.asarray(receiver_position), total_samples))


def convolve_moving(dry_list, rirs_list, positions_list) -> T.List[np.ndarray]:
    """Batched interpolate_moving_audio: for each i, dry (N,), RIRs (P, C, L), positions (P, 3)."""
    srcs = [MovingSource(d, r, trajectory_bounds(p, np.asarray(d).shape[-1]))
            for d, r, p in zip(dry_list, rirs_list, positions_list)]
    return default_renderer().render_host(srcs)


def render_scene(moving: T.Sequence[T.Tuple], static: T.Sequence[T.Tuple] = (), sr: float = 16000,
                 moving_lufs: T.Optional[float] = None, static_lufs: T.Optional[T.Sequence[float]] = None
                 ) -> T.Tuple[T.List[np.ndarray], T.List[np.ndarray]]:
    """One scene of SonicSet.process_single (SonicSet.py:77-101) in a single call:
    `moving` = [(dry (N,), rirs (P, C, L), positions (P, 3)), ...], `static` = [(dry (N,), rir (C, L)), ...].
    With `moving_lufs` (SonicSet uses -17) / `static_lufs` (SonicSet: [-24, -29] for noise, music) every
    stem is loudness-normalised like get_lufs_norm_audio: target ~ U(lufs - 2, lufs + 2) from the global
    NumPy RNG, drawn in the reference's order (all moving stems, then the static ones).
    Returns (moving stems, static stems), each (C, N) float32."""
    srcs: T.List = [MovingSource(d, r, trajectory_bounds(p, np.asarray(d).shape[-1])) for d, r, p in moving]
    srcs += [StaticSource(d, r) for d, r in static]
    targets = None
    if moving_lufs is not None or static_lufs is not None:
        targets = []
        for _ in moving:
            targets.append(None if moving_lufs is None else np.random.uniform(moving_lufs - 2, moving_lufs + 2))
        for i, _ in enumerate(static):
            l = None if static_lufs is None else static_lufs[i]
            targets.append(None if l is None else np.random.uniform(l - 2, l + 2))
    outs = default_renderer().render_host(srcs, lufs_targets=targets, sr=sr)
    return outs[: len(moving)], outs[len(moving):]


def render_mixtures(utterances: T.Sequence[dict], device: T.Optional[int] = None) -> T.List[dict]:
    """Whole path on the device, per utterance: render every speaker / noise stem, then assemble the training
    mixture exactly as the dataloader does (separation/look2hear/datas/movingdatamodule.py:105-124) without the
    stems leaving HBM.  Additive API (torch is used for device memory and copies only).

    utterance = {"speakers": [(dry (N,), rirs (P, C, L), positions (P, 3)), ...],     # speaker 0 is the reference
                 "noises":   [(dry (N,), rir (C, L)), ...],
                 "sirs": (S-1,) dB, "snr": dB}
    Returns per utterance {"mix": (C, N) float32, "speakers": (S, C, N) float32 (after their gains)}.
    Every stem of an utterance must have the same (C, N).  Each speaker's trajectory goes through trajectory_bounds,
    which draws from the global NumPy RNG like the reference, so identical calls give identical bits only from the
    same NumPy RNG state."""
    import torch
    from ._lib import SsMixItem
    R = default_renderer() if device is None else Renderer(device)
    dev = torch.device("cuda", R.device)
    lib = R.lib
    srcs, outs, plan = [], [], []
    for u in utterances:
        S, M = len(u["speakers"]), len(u["noises"])
        N = int(np.asarray(u["speakers"][0][0]).shape[-1])
        C = int(np.asarray(u["speakers"][0][1]).shape[1])
        for d, h, *_ in list(u["speakers"]) + list(u["noises"]):
            hs = np.asarray(h).shape
            if int(np.asarray(d).shape[-1]) != N or int(hs[-2]) != C:
                raise ValueError("render_mixtures: every stem of an utterance must have the same (C, N); got N=%d C=%d "
                                 "against N=%d C=%d" % (int(np.asarray(d).shape[-1]), int(hs[-2]), N, C))
        spk = torch.empty((S, C, N), dtype=torch.float32, device=dev)
        noi = torch.empty((M, C, N), dtype=torch.float32, device=dev)
        for i, (d, h, pos) in enumerate(u["speakers"]):
            b = trajectory_bounds(pos, N)
            srcs.append(MovingSource(torch.from_numpy(_as_f32(d).reshape(-1)).to(dev), torch.from_numpy(_as_f32(h)).to(dev),
                                     torch.from_numpy(b).to(dev), b))
            outs.append(spk[i])
        for i, (d, h) in enumerate(u["noises"]):
            srcs.append(StaticSource(torch.from_numpy(_as_f32(d).reshape(-1)).to(dev), torch.from_numpy(_as_f32(h)).to(dev)))
            outs.append(noi[i])
        plan.append((spk, noi, S, M, C, N, u))
    R.render_device(srcs, outs)
    n = len(plan)
    items = (SsMixItem * n)()
    keep = []
    nscr = int(lib.ss_mix_scratch_doubles())
    for k, (spk, noi, S, M, C, N, u) in enumerate(plan):
        mix = torch.empty((C, N), dtype=torch.float32, device=dev)
        sirs = torch.tensor(np.asarray(u.get("sirs", np.zeros(max(S - 1, 1))), dtype=np.float32).reshape(-1), device=dev)
        scr = torch.empty(nscr, dtype=torch.float64, device=dev)
        items[k] = SsMixItem(speakers=spk.data_ptr(), noises=noi.data_ptr(), sirs=sirs.data_ptr(), mix=mix.data_ptr(),
                             speakers_out=spk.data_ptr(), scratch=scr.data_ptr(), E=C * N, S=S, M=M,
                             snr=float(np.asarray(u.get("snr", 15.0)).reshape(-1)[0]))
        keep.append((mix, sirs, scr))
    _lib.check(lib.ss_mix_dev(R.ctx, items, n, ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    torch.cuda.synchronize(dev)
    return [{"mix": keep[k][0].cpu().numpy(), "speakers": plan[k][0].cpu().numpy()} for k in range(n)]
