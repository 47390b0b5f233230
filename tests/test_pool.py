"""Source pools (ss_pool; pooled slots ss_source.pool + pick_dev) on the CPU: the table a pooled slot is given holds the
blocks of every candidate at every start (pool_table_cap of ss_phases.cuh, exported by tests/emu/ss_emu_pool.cu,
against the table window_blocks finds for each candidate and start); k_blocks' clamp of a pick read from device memory
and the fields it writes into the slot; the ctypes mirror of ss_source against gcc; the exports; and the refusals that
need no device."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from emu import build_emu
from window_cases import B, _choice, _needs_numpy, _random_bounds
from sonicsim_b200 import _lib


@pytest.fixture(scope="module")
def emu_pool():
    return build_emu.load("ss_emu_pool")


def _cap(emu_pool, cands, aligned, L, wl, static=False):
    N = np.array([c[0] for c in cands], np.int32)
    P = np.array([c[1] for c in cands], np.int32)
    if static:
        return emu_pool.emu_pool_table_cap(None, None, N.ctypes.data, P.ctypes.data, len(cands), aligned, L, wl)
    off = np.cumsum([0] + [c[1] for c in cands[:-1]]).astype(np.int64)
    flat = np.ascontiguousarray(np.concatenate([c[2] for c in cands]), np.int32)
    return emu_pool.emu_pool_table_cap(flat.ctypes.data, off.ctypes.data, N.ctypes.data, P.ctypes.data, len(cands),
                                       aligned, L, wl)


def test_pool_table_cap_holds_every_candidate_at_every_start(emu_pool):
    """Pools of random trajectories with different P and N, L in {4096, 4097}, mixed aligned / grid choices: under the
    pool's blocking (aligned only if every candidate would choose it) the table holds window_blocks of every candidate
    at every start, and is the largest of them."""
    rng = np.random.default_rng(11)
    seen = set()
    for case in range(24):
        L = 4096 if case % 3 else 4097
        K = (L + B - 1) // B
        cands = []
        for _ in range(int(rng.integers(2, 6))):
            # odd cases: few long segments, which aligned blocking usually wins; even ones: any, some very short
            P = int(rng.integers(2, 6 if case % 2 else 24))
            N = int(rng.integers(max(P, 6000), 50000))
            b = _random_bounds(rng, P, N, short=case % 2 == 0 and bool(rng.integers(0, 3) == 0))
            cands.append((N, P, b))
        choices = [_choice(b, N, P, L) for N, P, b in cands]
        aligned = int(all(choices))
        seen.add((aligned, len(set(choices))))
        wl = int(rng.integers(1, min(c[0] for c in cands) + 1))
        need = max(int(_needs_numpy(N, b, aligned, K, wl).max()) for N, P, b in cands)
        assert _cap(emu_pool, cands, aligned, L, wl) == need, (case, aligned, wl)
        if aligned:
            # the same candidates on the grid (a pool that also holds a grid-choosing candidate)
            need_g = max(int(_needs_numpy(N, b, 0, K, wl).max()) for N, P, b in cands)
            assert _cap(emu_pool, cands, 0, L, wl) == need_g, (case, wl)
    assert (0, 2) in seen and any(a == 1 for a, _ in seen), seen       # mixed pools and all-aligned pools both ran


def test_pool_table_cap_of_static_pools(emu_pool):
    rng = np.random.default_rng(12)
    for L in (4096, 4097):
        K = (L + B - 1) // B
        cands = [(int(n), 1, None) for n in rng.integers(3 * B + 5, 60000, 5)]
        for wl in (1, B - 1, B, B + 1, 3 * B + 5, min(c[0] for c in cands)):
            need = max(int(_needs_numpy(N, None, 0, K, wl).max()) for N, _, _ in cands)
            assert _cap(emu_pool, cands, 0, L, wl, static=True) == need, (L, wl)


def test_clamp_of_a_device_pick(emu_pool):
    bad = ctypes.c_int32()
    for v, n, want, flagged in [(0, 1, 0, 0), (0, 5, 0, 0), (4, 5, 4, 0), (5, 5, 4, 1), (-1, 5, 0, 1),
                                (-(1 << 31), 5, 0, 1), ((1 << 31) - 1, 5, 4, 1), (3, 1 << 24, 3, 0),
                                ((1 << 24), 1 << 24, (1 << 24) - 1, 1)]:
        assert (emu_pool.emu_clamp_pick(v, n, ctypes.byref(bad)), bad.value) == (want, flagged), (v, n)


def test_pick_writes_the_candidate_into_the_slot(emu_pool):
    out = np.zeros(10, np.int32)
    for N, P, C, K, direct in [(20000, 40, 6, 1, 0), (4097, 3, 2, 2, 1), (1, 1, 5, 1, 1), (4096, 1, 1, 1, 0)]:
        emu_pool.emu_pick_candidate(N, P, C, K, direct, out.ctypes.data)
        assert out[:5].tolist() == [N, P, (N + B - 1) // B, 0, P * C * K]
        assert out[5:].tolist() == [1, 1, 1, direct, 1], (N, P, direct)


def test_ss_source_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sonicsim_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(ss_source));']
    for fname, _ in _lib.SsSource._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(ss_source, %s));' % (fname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {l.split()[0]: int(l.split()[1]) for l in out if l.strip()}
    assert got["size"] == ctypes.sizeof(_lib.SsSource)
    for fname, _ in _lib.SsSource._fields_:
        assert got[fname] == getattr(_lib.SsSource, fname).offset, fname
    assert [f for f, _ in _lib.SsSource._fields_][-2:] == ["pool", "pick_dev"]


def test_pool_symbols_are_exported():
    lib = ctypes.CDLL(_lib.build())
    for name in ("ss_pool_create", "ss_pool_bytes", "ss_pool_destroy"):
        assert hasattr(lib, name) and name in _lib.EXPORTS, name
    assert lib.ss_version() >= 106
    assert _lib.load().ss_pool_bytes(None) == 0


def test_debug_plan_refuses_a_pooled_slot():
    """ss_debug_plan plans one source on the host; a pooled slot's candidate is only known on the device."""
    lib = _lib.load()
    b = np.array([0, 5000, 10000], np.int32)
    out = np.zeros((16, 4), np.int32)
    for field in ("pool", "pick_dev"):
        item = _lib.SsSource(x=1, rir=1, out=1, bounds=b.ctypes.data, N=10000, P=3, C=2, L=300,
                             mode=_lib.SS_MOVING_BOUNDS, bounds_host=b.ctypes.data, win_start=0, win_len=100)
        assert lib.ss_debug_plan(ctypes.byref(item), out.ctypes.data, 16, None) > 0
        setattr(item, field, 4096)
        assert lib.ss_debug_plan(ctypes.byref(item), out.ctypes.data, 16, None) == _lib.SS_ERR_INVALID, field


def test_python_refuses_pooled_slots_off_plans():
    from sonicsim_b200 import render
    slot = render.Pooled(object(), object(), (0, 10))
    for where in ("plan_host", "render_device"):
        with pytest.raises(ValueError, match="pooled"):
            render._refuse_pooled([render.StaticSource(None, None), slot], where)
    render._refuse_pooled([render.StaticSource(None, None)], "plan_host")
