"""Tap-form host banks (SS_BANK_TAPS) on the CPU, through the kernels' own helpers (exported by tests/emu/ss_emu_taps.cu):
  - the stored rows of a tap bank are the RIR taps zero-padded to K * 4096, divided by the abs-max with normalisation (an
    all-zero RIR set is stored undivided), and its cut table is the spectral bank's;
  - k_prepare's CTAs over tap_source, at the plan-time CTA count, turn the staged rows [row0, row0 + rows) of any read
    set (stage_set) into spectra bit-equal to the matching rows of the spectral bank of the same RIRs, in both sets; the
    CTAs past the run's row pairs write nothing, and rows outside the staged set (NaN) are never read;
  - the staging area a plan carves for a slot (stage_area) adds stage_cap rows * 16 KB of taps behind a spectral slot's
    unchanged regions, every region 256-byte aligned and large enough for the rows and samples any run stages (rows *
    16 KB of taps against sets * rows * 32 KB of spectra); the block behind the areas (tap_block: StageTaps, transform
    Sources, CTA prefix, zero word) holds each part without overlap."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from oracle import sonicsim_oracle as so
from window_cases import B, KSPEC, _k, _p, _random_bounds


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_taps")


def _tap_bank(emu, h, normalize, taps):
    P, C, L = h.shape
    rows = np.full((P * C * _k(L), B), np.nan, np.float32)
    cut = np.zeros(P * C, np.int32) if taps else None
    emu.emu_tap_bank(_p(h), P, C, L, int(normalize), taps, _p(rows), _p(cut))
    return rows, cut


def _spec_bank(emu, h, normalize, taps):
    P, C, L = h.shape
    sets = 2 if taps else 1
    spec = np.full((sets * P * C * _k(L), KSPEC), np.nan, np.complex64)
    cut = np.zeros(P * C, np.int32) if taps else None
    emu.emu_bank_create(_p(h), P, C, L, int(normalize), taps, _p(spec), _p(cut))
    return spec, cut


def _rirs(rng, P, C, L):
    h = np.ascontiguousarray(so.synth_rirs(rng, P, C, L), np.float32)
    return np.ascontiguousarray(h * np.float32(0.37))          # abs-max != 1: normalisation divides


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("K", [1, 2, 3])
@pytest.mark.parametrize("whole", [True, False])
@pytest.mark.parametrize("P", [1, 3])
@pytest.mark.parametrize("normalize", [False, True])
@pytest.mark.parametrize("taps", [0, 40])
def test_tap_bank_rows_are_the_padded_divided_taps(emu, K, whole, P, normalize, taps):
    rng = np.random.default_rng(K * 100 + P * 10 + normalize * 3 + (taps > 0))
    C = 2
    L = K * B if whole else (K - 1) * B + 1 + int(rng.integers(0, B - 1))
    h = _rirs(rng, P, C, L)
    rows, cut = _tap_bank(emu, h, normalize, taps)
    want = h / np.max(np.abs(h)) if normalize else h                # float32 / float32: IEEE division, as div_rn
    pad = np.zeros((P, C, K * B), np.float32)
    pad[:, :, :L] = want
    assert np.array_equal(_bits(rows), _bits(pad.reshape(P * C * K, B)))
    if taps:
        _, cut_spec = _spec_bank(emu, h, normalize, taps)
        assert np.array_equal(cut, cut_spec)


def test_all_zero_rir_set_is_stored_undivided(emu):
    h = np.zeros((2, 2, B + 300), np.float32)
    h[0, 1, 7] = -0.0                                                # a -0 divided by m = 0 would be NaN
    h[1, 0, :] = -0.0
    rows, cut = _tap_bank(emu, h, True, 16)
    pad = np.zeros((2, 2, 2 * B), np.float32)
    pad[:, :, :h.shape[2]] = h
    assert np.array_equal(_bits(rows), _bits(pad.reshape(-1, B)))
    _, cut_spec = _spec_bank(emu, h, True, 16)
    assert np.array_equal(cut, cut_spec)


class Cand:
    """One candidate: trajectory (None: static), RIRs, its spectral bank and its tap bank (normalised or not, with a
    direct set when taps > 0)."""

    def __init__(self, emu, rng, N, P, C, L, normalize, taps):
        self.N, self.P, self.C, self.L, self.K = N, P, C, L, _k(L)
        self.bounds = None if P == 1 else _random_bounds(rng, P, N, False)
        h = _rirs(rng, P, C, L)
        self.spec, self.cut = _spec_bank(emu, h, normalize, taps)
        self.rows, tcut = _tap_bank(emu, h, normalize, taps)
        assert (tcut is None and self.cut is None) or np.array_equal(tcut, self.cut)
        self.sets = 2 if taps else 1

    def stage_set(self, emu, ws, wl):
        out = np.zeros(4, np.int32)
        emu.emu_stage_set(self.N, self.P, self.C, self.K, _p(self.bounds), ws, wl, _p(out))
        return [int(v) for v in out]


def _cap(emu, c, wl):
    out = np.zeros(2, np.int32)
    N, P, K = (np.array([v], np.int32) for v in (c.N, c.P, c.K))
    if c.bounds is None:
        emu.emu_stage_cap(None, None, _p(N), _p(P), _p(K), 1, c.C, wl, _p(out))
    else:
        emu.emu_stage_cap(_p(c.bounds), _p(np.zeros(1, np.int64)), _p(N), _p(P), _p(K), 1, c.C, wl, _p(out))
    return int(out[0])


def _cap_nx(emu, c, wl):
    out = np.zeros(2, np.int32)
    N, P, K = (np.array([v], np.int32) for v in (c.N, c.P, c.K))
    emu.emu_stage_cap(_p(c.bounds), None if c.bounds is None else _p(np.zeros(1, np.int64)), _p(N), _p(P), _p(K), 1,
                      c.C, wl, _p(out))
    return int(out[0]), int(out[1])


def _transform(emu, c, row0, rows, cap):
    staged = np.full_like(c.rows, np.nan)                            # the staged rows, NaN everywhere else
    staged[row0:row0 + rows] = c.rows[row0:row0 + rows]
    spec = np.full((c.sets * cap, 2 * KSPEC), np.nan, np.float32).view(np.complex64)
    info = np.zeros(5, np.int32)
    emu.emu_tap_transform(_p(staged), _p(c.cut), c.P, c.C, c.K, row0, rows, c.sets, cap, _p(spec), _p(info))
    return spec, [int(v) for v in info]


# (N, P, C, L, normalize, direct taps, window): static and moving, K = 1..3, an odd P * C * K (3 * 1 * 3 = 9, 1 * 3 * 1)
CASES = [(40000, 1, 3, 3000, False, 0, 5000),
         (40000, 1, 2, 2 * B + 17, True, 30, 7000),
         (60000, 3, 1, 3 * B, True, 0, 9000),
         (60000, 5, 2, B + 900, False, 25, 4000),
         (60000, 4, 2, 4000, True, 25, 12000)]


@pytest.mark.parametrize("case", CASES, ids=["static_k1_odd", "static_k3_direct_norm", "moving_k3_odd_norm",
                                             "moving_k2_direct", "moving_k1_direct_norm"])
def test_transform_of_staged_rows_equals_the_spectral_bank(emu, case):
    N, P, C, L, normalize, taps, wl = case
    rng = np.random.default_rng(N + P + L)
    c = Cand(emu, rng, N, P, C, L, normalize, taps)
    cap = _cap(emu, c, wl)
    last = N - wl
    starts = {0, last, last // 2, min(last, (c.K + 2) * B)} | {int(v) for v in rng.integers(0, last + 1, 6)}
    for b in ([] if c.bounds is None else c.bounds[1:-1]):
        starts |= {int(v) for v in (b - 1, b, b + 1) if 0 <= v <= last}
    rows_h = P * C * c.K
    seen_rows = set()
    for ws in sorted(starts):
        _, _, row0, rows = c.stage_set(emu, ws, wl)
        assert row0 % 2 == 0 and rows <= cap and row0 + rows <= rows_h
        spec, info = _transform(emu, c, row0, rows, cap)
        pairs = c.sets * ((rows + 1) // 2)
        ctas = c.sets * ((cap + 1) // 2)
        assert info == [pairs, pairs, ctas - pairs, rows, row0], (ws, info)
        for s in range(c.sets):
            got = spec[s * rows:(s + 1) * rows]
            want = c.spec[s * rows_h + row0:s * rows_h + row0 + rows]
            assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (ws, s, row0, rows)
        assert np.isnan(spec[c.sets * rows:].view(np.float32)).all()   # the extra CTAs and the unused cap: untouched
        seen_rows.add((row0, rows))
    assert len(seen_rows) > 1 or P == 1


def _area(emu, sets, rows_cap, nx, taps):
    out = np.zeros(5, np.int64)
    emu.emu_stage_area(sets, rows_cap, nx, int(taps), _p(out))
    return [int(v) for v in out]


def test_staging_area_and_tap_block(emu):
    rng = np.random.default_rng(5)
    for taps in (0, 20):
        c = Cand(emu, rng, 60000, 6, 2, 2 * B, False, taps)
        wl = 8000
        cap, nx = _cap_nx(emu, c, wl)
        spec_area = _area(emu, c.sets, cap, nx, False)
        view, spec, x, tap, end = _area(emu, c.sets, cap, nx, True)
        assert [view, spec, x, tap] == spec_area[:4] and spec_area[4] == tap   # the spectral slot's regions, unchanged
        assert all(v % 256 == 0 for v in (view, spec, x, tap, end))
        assert spec - view >= 56 and x - spec >= c.sets * cap * KSPEC * 8 and tap - x >= 4 * nx
        assert end - tap == cap * B * 4                                  # stage_cap rows of taps, 16 KB each
        for ws in (0, 20000, 60000 - wl):
            xa, xb, row0, rows = c.stage_set(emu, ws, wl)
            assert rows <= cap and ((xb + 3) & ~3) - (xa & ~3) <= nx
            assert rows * B * 4 * 2 * c.sets == c.sets * rows * KSPEC * 8  # taps staged: half (quarter) the spectra
    sizes = np.zeros(2, np.int64)
    for at, n_staged, n_tap in ((0, 1, 1), (12345, 7, 3), (1 << 20, 65535, 65535), (256, 40, 1)):
        out = np.zeros(5, np.int64)
        emu.emu_tap_block(at, n_staged, n_tap, _p(out), _p(sizes))
        taps, src, prefix, zero, end = (int(v) for v in out)
        assert all(v % 256 == 0 for v in (taps, src, prefix, zero, end)) and at <= taps < at + 256
        assert src - taps >= n_staged * int(sizes[0]) and prefix - src >= n_tap * int(sizes[1])
        assert zero - prefix >= 4 * (n_tap + 1) and end - zero >= 4


def test_python_and_c_refusals_without_a_device():
    from sonicsim_b200 import _lib, render
    lib = _lib.load()
    assert "ss_bank_flags" in _lib.EXPORTS and lib.ss_bank_flags(None) == 0
    assert _lib.SS_BANK_TAPS == 0x200
    assert lib.ss_version() == 108

    class R:
        ctx, device = ctypes.c_void_p(1000), 0

    h = np.zeros((2, B), np.float32)
    with pytest.raises(ValueError, match="needs host=True"):
        render.Renderer.rir_bank(R, h, form="taps")
    with pytest.raises(ValueError, match="form must be 'spectra' or 'taps'"):
        render.Renderer.rir_bank(R, h, host=True, form="halfspectra")
