"""Start draws of device plans (ss_plan_draw) and level tables of pools (ss_pool_levels) on the CPU: the per-try
functions k_draw runs (draw_span, draw_start, draw_silent of ss_phases.cuh, exported by tests/emu/ss_emu_draw.cu)
against tests/draw_reference.py and against the starts the unmodified dataloader loop chose (tests/golden/crop_draw.npz);
the ctypes mirror of ss_plan_draw against gcc; the exports."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from emu import build_emu
import draw_reference as dr
from sonicsim_b200 import _lib

GOLDEN = os.path.join(ROOT, "tests", "golden", "crop_draw.npz")


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_draw")


def emu_draw(emu, tables, D, reader_N, length, u, thr=-40.0):
    tabs = [np.ascontiguousarray(t, np.float64) for t in tables]
    ptrs = (ctypes.c_void_p * len(tabs))(*[t.ctypes.data for t in tabs])
    Da = np.ascontiguousarray(D, np.float64)
    Na = np.ascontiguousarray(reader_N, np.int32)
    ua = np.ascontiguousarray(u, np.float64)
    used = ctypes.c_int32()
    s = emu.emu_draw(ctypes.cast(ptrs, ctypes.c_void_p), Da.ctypes.data, len(tabs), Na.ctypes.data, len(Na), length,
                     ua.ctypes.data, len(ua), thr, ctypes.byref(used))
    return s, used.value


def test_golden_starts_of_the_dataloader_loop(emu):
    """The unmodified :81-99 on float32 speakers with silent stretches: first try, only try 100, every try silent, S = 1,
    2, 3, mono and channels.  The restatement and the kernel's per-try functions choose the same start and try."""
    g = np.load(GOLDEN)
    names = [str(v) for v in g["names"]]
    assert {"first_try", "only_try_100", "all_silent"} <= set(names)
    length = int(g["len"])
    seen_S, seen_used = set(), set()
    for k in range(int(g["n_cases"])):
        wav, u = g["wav%d" % k], g["u%d" % k]
        want = (int(g["start%d" % k]), int(g["used%d" % k]))
        mono = wav.ndim == 2
        tabs = [dr.level_table(wav[s][None] if mono else wav[s], mono) for s in range(wav.shape[0])]
        D = [length if mono else wav.shape[1] * length] * wav.shape[0]
        N = [wav.shape[-1]] * wav.shape[0]
        assert dr.draw(tabs, D, N, length, u) == want, names[k]
        assert emu_draw(emu, tabs, D, N, length, u) == want, names[k]
        seen_S.add(wav.shape[0])
        seen_used.add(want[1])
    assert {1, 2, 3} <= seen_S and {0, 1, 101} <= seen_used


def test_start_mapping(emu):
    """min(floor(u * M), M - 1): M = 1, u = 0 and u = 1 - 2^-53 (the largest u below 1), u = 1 and beyond, negative, NaN."""
    top = 1.0 - 2.0 ** -53
    for M in (1, 2, 3, 7, 1000, 65536, 480001, (1 << 31) - 1):
        assert emu.emu_draw_start(0.0, M) == 0 == dr.start_of(0.0, M)
        assert emu.emu_draw_start(top, M) == M - 1 == dr.start_of(top, M)
        for u in (1.0, 1.5, float("inf")):
            assert emu.emu_draw_start(u, M) == M - 1 == dr.start_of(u, M), (u, M)
        for u in (-0.25, -float("inf"), float("nan")):
            assert emu.emu_draw_start(u, M) == 0 == dr.start_of(u, M), (u, M)
    rng = np.random.default_rng(3)
    for _ in range(2000):
        M, u = int(rng.integers(1, 1 << 20)), float(rng.random())
        assert emu.emu_draw_start(u, M) == dr.start_of(u, M) == min(int(np.floor(u * M)), M - 1)


def _gappy(rng, N, C=1):
    """A stem with silent stretches of random length, dataloader-like."""
    y = (0.05 * rng.standard_normal((C, N))).astype(np.float32)
    pos = 0
    while pos < N:
        g = int(rng.integers(0, N // 3))
        y[:, pos:pos + g] = 0
        pos += g + int(rng.integers(N // 10, N // 3))
    return y


def test_seeded_draws_against_the_reference(emu):
    """Random pools of speakers with gaps, readers of different N (the shortest need not be a speaker), M = 1, 8
    speakers, 4096 tries and tries that all fail: the emulated draw equals the restatement."""
    rng = np.random.default_rng(5)
    seen = set()
    for case in range(160):
        mono = case % 2 == 0
        C = 1 if mono else int(rng.integers(1, 4))
        S = 8 if case % 10 == 3 else int(rng.integers(1, 4))
        length = int(rng.integers(50, 400))
        tries = 4096 if case % 10 == 5 else int(rng.integers(1, 120))
        Ns = [int(rng.integers(length, 3 * length)) for _ in range(S)]
        extra = [int(rng.integers(length, 3 * length)) for _ in range(int(rng.integers(0, 3)))]
        if case % 10 == 7:
            extra.append(length)                               # M = 1: a reader as long as the crop
        tabs = [dr.level_table(_gappy(rng, n, C), mono) for n in Ns]
        D = [length * (1 if mono else C)] * S
        u = rng.random(tries)
        thr = -40.0 if case % 4 else -25.0
        want = dr.draw(tabs, D, Ns + extra, length, u, thr)
        if dr.margins(tabs, D, Ns + extra, length, u, thr) < 1e-9:
            continue
        assert emu_draw(emu, tabs, D, Ns + extra, length, u, thr) == want, case
        seen.add(("M1" if min(Ns + extra) == length else "") + ("pass" if want[1] else "fail"))
        if S == 8:
            seen.add("S8")
        if tries == 4096:
            seen.add("4096")
    assert {"pass", "fail", "M1pass", "S8", "4096"} <= seen, seen


def test_level_exactly_at_the_threshold_is_not_silent(emu):
    """10 log10(1e-4) is exactly -40 (and 10 log10(1) exactly 0): a crop at the threshold passes."""
    length = 4
    for ms, thr in ((1e-4, -40.0), (1.0, 0.0)):
        Q = np.arange(0, 11, dtype=np.float64) * ms              # e[n] = ms: mean square ms over any crop
        assert dr.level_db(Q, 0, length, length) == thr
        for u0 in (0.0, 0.5):
            assert emu_draw(emu, [Q], [length], [10], length, [u0], thr)[1] == 1
            assert dr.draw([Q], [length], [10], length, [u0], thr)[1] == 1
        # a hair below: silent at every try, the last try's start is kept
        Qb = Q * (1 - 1e-12)
        assert emu_draw(emu, [Qb], [length], [10], length, [0.0, 0.9], thr) == (6, 0)
        assert dr.draw([Qb], [length], [10], length, [0.0, 0.9], thr) == (6, 0)


def test_level_tables_restated():
    """The NumPy level table: mono terms fold the channels in order before squaring; channel terms sum the squares."""
    rng = np.random.default_rng(9)
    y = rng.standard_normal((3, 1000)).astype(np.float32)
    v = ((y[0] + y[1]).astype(np.float32) + y[2]).astype(np.float32) / np.float32(3)
    Qm = dr.level_table(y, True)
    assert Qm[0] == 0 and Qm.shape == (1001,)
    assert np.allclose(np.diff(Qm), (v * v).astype(np.float64), rtol=0, atol=1e-13 * Qm[-1])
    Qc = dr.level_table(y, False)
    assert np.allclose(np.diff(Qc), (y.astype(np.float64) ** 2).sum(0), rtol=1e-6, atol=1e-13 * Qc[-1])


def test_ss_plan_draw_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sonicsim_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(ss_plan_draw));']
    for fname, _ in _lib.SsPlanDraw._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(ss_plan_draw, %s));' % (fname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {l.split()[0]: int(l.split()[1]) for l in out if l.strip()}
    assert got["size"] == ctypes.sizeof(_lib.SsPlanDraw)
    for fname, _ in _lib.SsPlanDraw._fields_:
        assert got[fname] == getattr(_lib.SsPlanDraw, fname).offset, fname


def test_draw_symbols_are_exported():
    lib = ctypes.CDLL(_lib.build())
    for name in ("ss_pool_levels", "ss_pool_level_table", "ss_plan_create_ex"):
        assert hasattr(lib, name) and name in _lib.EXPORTS, name
    assert lib.ss_version() >= 107
    L = _lib.load()
    assert L.ss_pool_levels(None, 0) == _lib.SS_ERR_INVALID
    assert L.ss_pool_level_table(None, 0) is None
