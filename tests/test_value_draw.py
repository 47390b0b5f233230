"""Value draws (ss_value_draw; render.ValueDraw) on the CPU, through k_values' own code (ss_phases.cuh: value_word,
value_f64, value_f32 and value_row, exported by tests/emu/ss_emu_values.cu).
  - Emulated rows equal the NumPy restatement of tests/value_reference.py bit for bit over many (seed, t, r, b), for
    float32, float64, int32 and distinct draws, k = 1, 2, 3, 64 and 4096, base / stride chains, and any lane split.
  - Extreme words: x = 2^64 - 1 gives values below high, in float32 (low = -6, high = 6 included), float64 and int32
    with high - low = 2^31 - 1 and 2^32 - 1; x = 0 gives low.
  - Distributions within 5 standard errors or by a chi-square test: uniform reals (mean, variance, bin counts),
    integers over small and large ranges, distinct samples of 2 from 3 (all 6 ordered pairs, never a repeat), and 101
    tries of u independent across elements.
  - The value blocks and the layout blocks are disjoint for every r below the bounds.
  - render.ValueDraw's structural refusals are ValueErrors raised before any tensor or C call.
The plan-level refusals and the kernel itself need a device: tests/test_gpu_value_draw.py."""
import numpy as np
import pytest
from scipy import stats

import value_reference as vr
from value_reference import Spec

SEEDS = [(0, 0), (20261018, 7), (-77, 123456789), ((1 << 63) - 1, -1), (-(1 << 63), 1 << 40)]


@pytest.fixture(scope="module")
def emu():
    return vr.load_emu()


def assert_bits(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape
        assert np.array_equal(g.view(np.uint8), w.view(np.uint8))


def test_words_follow_the_stream(emu):
    for seed, t in SEEDS:
        for r in (0, 1, 5, (1 << 20) - 1):
            for b in (0, 1, 65534):
                for j in (0, 1, 2, 3, 4094, 4095):
                    assert emu.emu_value_word(seed, t, r, b, j) == vr.word(seed, t, r, b, j), (seed, t, r, b, j)


CHAINS = [
    [Spec(np.float32, 1, -6, 6), Spec(np.float64, 3, 10, 20), Spec(np.int32, 2, 0, 7)],
    [Spec(np.int32, 1, 0, 5), Spec(np.int32, 3, 0, 3, distinct=True, base=0, stride=3), Spec(np.float32, 2, -6, 6),
     Spec(np.float32, 1, 10, 20), Spec(np.float64, 101)],
    [Spec(np.int32, 1, 2, 9, distinct=True), Spec(np.int32, 64, -5, 1000, distinct=True, base=0, stride=1000),
     Spec(np.int32, 1, 0, 4, base=0, stride=2), Spec(np.int32, 2, -(1 << 31), (1 << 31) - 1)],
    [Spec(np.float64, 64, -19, -15), Spec(np.float32, 64, 0.25, 0.5), Spec(np.int32, 64, 0, 64, distinct=True)],
    [Spec(np.float64, 4096, -1e300, 1e300), Spec(np.float32, 4096, -2, 3), Spec(np.int32, 4096, -3, 40000)],
]


@pytest.mark.parametrize("chain", range(len(CHAINS)))
def test_emulated_rows_equal_the_restatement(emu, chain):
    specs = CHAINS[chain]
    nrows = 2 if max(s.k for s in specs) > 100 else 5
    for seed, t in SEEDS:
        want = vr.rows(specs, nrows, seed, t)
        assert_bits(vr.emu_rows(emu, specs, nrows, seed, t), want)
        assert_bits(vr.emu_rows(emu, specs, nrows, seed, t, lanes=1), want)       # any lane split: the same values
        assert_bits(vr.emu_rows(emu, specs, nrows, seed, t, lanes=7), want)
        for s, o in zip(specs, want):
            if s.base is None:
                assert (o >= s.low).all() and (o < s.high).all()
            if s.distinct:
                assert all(len(set(row)) == s.k for row in o.tolist())
    assert not all(np.array_equal(a, b) for a, b in zip(vr.emu_rows(emu, specs, nrows, 1, 2),
                                                        vr.emu_rows(emu, specs, nrows, 1, 3)))


def test_base_chains_add_the_base_times_stride(emu):
    specs = [Spec(np.int32, 1, 0, 1000), Spec(np.int32, 3, 0, 3, distinct=True, base=0, stride=3),
             Spec(np.int32, 1, 0, 3, distinct=True), Spec(np.int32, 4, 10, 20, base=2, stride=100)]
    scene, picks, d, v = vr.emu_rows(emu, specs, 500, 4, 9)
    assert ((picks - scene * 3) >= 0).all() and ((picks - scene * 3) < 3).all()
    assert (np.sort(picks - scene * 3, axis=1) == [0, 1, 2]).all()
    off = v - d * 100
    assert ((off >= 10) & (off < 20)).all()


def test_extreme_words(emu):
    top = (1 << 64) - 1
    for low, high in [(-6, 6), (10, 20), (0, 1), (-19, -15), (-1e-30, 1e-30), (1, 1 + 2 ** -20), (-2 ** 100, 2 ** 100)]:
        f = emu.emu_value_f32(low, high, top)
        assert np.float32(f) < np.float32(high) and f >= low and f == vr.real32(top, low, high), (low, high)
        assert emu.emu_value_f32(low, high, 0) == np.float32(low)
    for low, high in [(-6, 6), (0, 1), (10, 20), (1, 1 + 2 ** -50), (-1e300, 1e300)]:
        f = emu.emu_value_f64(low, high, top)
        assert f < high and f >= low and f == vr.real64(top, low, high), (low, high)
        assert emu.emu_value_f64(low, high, 0) == low
    # a result that rounds up to high is the largest value below it
    assert emu.emu_value_f64(1, 1 + 2 ** -50, top) == np.nextafter(1 + 2 ** -50, 0)
    assert emu.emu_value_f32(1, 1 + 2 ** -20, top) == np.nextafter(np.float32(1 + 2 ** -20), np.float32(0))
    for n in (1, 3, (1 << 31) - 1, (1 << 32) - 1):
        assert emu.emu_value_below(top, n) == n - 1
        assert emu.emu_value_below(0, n) == 0
    # int32 draws over [-2^31 + 1, 2^31 - 1) hit their ends: rows of one (seed, t), checked against the restatement
    specs = [Spec(np.int32, 1, -(1 << 31) + 1, (1 << 31) - 1), Spec(np.int32, 1, -(1 << 31), (1 << 31) - 1)]
    assert_bits(vr.emu_rows(emu, specs, 3, 5, 5), vr.rows(specs, 3, 5, 5))


# ---------------------------------------------------------------------------------------------------- distributions
def draws(emu, spec, n=20000, seed=11, t=3):
    return vr.emu_rows(emu, [spec], n, seed, t)[0]


@pytest.mark.parametrize("dtype,low,high", [(np.float64, 0, 1), (np.float64, -19, -15), (np.float32, -6, 6),
                                            (np.float32, 10, 20)])
def test_uniform_reals(emu, dtype, low, high):
    x = draws(emu, Spec(dtype, 8, low, high)).astype(np.float64).ravel()
    n, w = x.size, high - low
    mean_se = w * np.sqrt(1 / 12 / n)
    assert abs(x.mean() - (low + high) / 2) < 5 * mean_se
    var = w * w / 12
    var_se = np.sqrt((w ** 4 / 80 - var * var) / n)
    assert abs(x.var() - var) < 5 * var_se
    counts = np.histogram(x, bins=20, range=(low, high))[0]
    assert stats.chisquare(counts).pvalue > 1e-4
    assert (x >= low).all() and (x < high).all()


@pytest.mark.parametrize("low,high", [(0, 3), (-6, 7), (0, 101), (0, 1 << 30), (-(1 << 31), (1 << 31) - 1)])
def test_uniform_integers(emu, low, high):
    x = draws(emu, Spec(np.int32, 4, low, high)).astype(np.int64).ravel()
    assert (x >= low).all() and (x < high).all()
    n = high - low
    if n <= 200:
        counts = np.bincount(x - low, minlength=n)
        assert stats.chisquare(counts).pvalue > 1e-4
    else:                                                  # large ranges: 16 equal bins of the offset
        counts = np.bincount(((x - low) * 16) // n, minlength=16)
        assert stats.chisquare(counts).pvalue > 1e-4
        mean_se = n * np.sqrt(1 / 12 / x.size)
        assert abs(x.mean() - (low + high - 1) / 2) < 5 * mean_se


def test_distinct_pairs_of_three(emu):
    x = draws(emu, Spec(np.int32, 2, 1, 4, distinct=True), n=30000)
    assert (x[:, 0] != x[:, 1]).all()
    pairs = (x[:, 0] - 1) * 3 + (x[:, 1] - 1)
    counts = np.bincount(pairs, minlength=9)
    assert counts[[0, 4, 8]].sum() == 0                    # never a repeat
    six = counts[[1, 2, 3, 5, 6, 7]]
    assert stats.chisquare(six).pvalue > 1e-4
    p = 1 / 6
    assert (np.abs(six / x.shape[0] - p) < 5 * np.sqrt(p * (1 - p) / x.shape[0])).all()


def test_distinct_samples_are_uniform_permutations(emu):
    x = draws(emu, Spec(np.int32, 3, 0, 5, distinct=True), n=12000, seed=3)
    assert all(len(set(r)) == 3 for r in x.tolist())
    code = x[:, 0] * 25 + x[:, 1] * 5 + x[:, 2]
    counts = np.unique(code, return_counts=True)[1]
    assert counts.size == 60 and stats.chisquare(counts).pvalue > 1e-4


def test_crop_variates_are_independent_across_tries(emu):
    u = draws(emu, Spec(np.float64, 101), n=8000, seed=5, t=77)
    c = np.corrcoef(u.T)
    off = c[~np.eye(101, dtype=bool)]
    assert np.abs(off).max() < 5 / np.sqrt(u.shape[0])
    # consecutive tries share Philox blocks two by two: their joint 4 x 4 cells are uniform
    for j in (0, 1, 99):
        cells = (np.floor(u[:, j] * 4) * 4 + np.floor(u[:, j + 1] * 4)).astype(int)
        assert stats.chisquare(np.bincount(cells, minlength=16)).pvalue > 1e-4


def test_rows_and_counters_differ(emu):
    spec = Spec(np.float64, 4)
    a = vr.emu_rows(emu, [spec, spec], 64, 9, 1)
    b = vr.emu_rows(emu, [spec, spec], 64, 9, 2)
    c = vr.emu_rows(emu, [spec, spec], 64, 10, 1)
    assert not np.array_equal(a[0], a[1])                  # draws r = 0 and 1: other blocks
    assert len(np.unique(a[0])) == a[0].size               # rows and elements: other values
    assert not np.array_equal(a[0], b[0]) and not np.array_equal(a[0], c[0])


# ---------------------------------------------------------------------------------------------------- stream layout
def test_value_blocks_and_layout_blocks_are_disjoint():
    # a layout draw r takes c1 = r, r < 2^31; a value draw r < 2^20 takes c1 = 2^31 | r << 11 | j >> 1, j < 4096
    r = np.arange(1 << 20, dtype=np.uint64)
    for h in (0, 1, 2046, 2047):
        c1 = (np.uint64(1 << 31) | r << np.uint64(11) | np.uint64(h)).astype(np.uint64)
        assert (c1 >= (1 << 31)).all() and (c1 < (1 << 32)).all()          # never a layout block's c1
        assert ((c1 >> np.uint64(11)) & np.uint64((1 << 20) - 1) == r).all()  # r and j >> 1 read back: one block each
        assert (c1 & np.uint64(2047) == h).all()
    assert vr.word(1, 2, (1 << 20) - 1, 3, 4095) != vr.word(1, 2, (1 << 20) - 1, 3, 4094)


# ---------------------------------------------------------------------------------------------------- refusals
def test_value_draw_structural_refusals_before_any_c_call():
    import torch
    from sonicsim_b200 import render
    R = object.__new__(render.Renderer)                    # no context: a refusal must come before any C call
    R.device, R.lib = 0, None
    cpu = torch.zeros(4, dtype=torch.float32)
    with pytest.raises(ValueError, match="must be a ValueDraw"):
        R._device_values([("out", "rng")], [], (None,) * 5, [])
    with pytest.raises(ValueError, match="CUDA"):
        R._device_values([render.ValueDraw(cpu, cpu)], [], (None,) * 5, [])
    with pytest.raises(ValueError, match="float32, float64 or int32"):
        R._device_values([render.ValueDraw(torch.zeros(4, dtype=torch.int64), cpu)], [], (None,) * 5, [])
    with pytest.raises(ValueError, match="2\\^20"):
        R._device_values([None] * ((1 << 20) + 1), [], (None,) * 5, [])
