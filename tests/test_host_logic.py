"""Host-side logic of the package (no GPU): the trajectory setup mirror, argument handling, and
that the C-ABI library loads and exports every symbol include/sonicsim_b200.h declares."""
import ctypes
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from sonicsim_b200 import SonicSim_moving as sm
from sonicsim_b200 import _lib


def test_setup_dynamic_interp_bit_exact_vs_reference_golden(golden):
    g = golden("setup_dynamic_interp")
    for k in range(int(g["n_cases"])):
        np.random.seed(int(g[f"seed{k}"]))
        idx, w = sm.setup_dynamic_interp(g[f"pos{k}"], int(g[f"N{k}"]))
        assert idx.dtype == np.int64 and w.dtype == np.float32
        assert np.array_equal(idx, g[f"idx{k}"]) and np.array_equal(w, g[f"w{k}"])


def test_bounds_are_the_compact_form(golden):
    g = golden("setup_dynamic_interp")
    for k in range(int(g["n_cases"])):
        np.random.seed(int(g[f"seed{k}"]))
        spi = sm._samples_per_interval(g[f"pos{k}"], int(g[f"N{k}"]))
        b = sm.bounds_from_counts(spi)
        assert b.dtype == np.int32 and b[0] == 0 and b[-1] == int(g[f"N{k}"]) and len(b) == len(g[f"pos{k}"])
        assert np.array_equal(np.repeat(np.arange(len(spi)), spi), g[f"idx{k}"])


def test_degenerate_path_raises_value_error():
    with np.errstate(all="ignore"):
        with pytest.raises(ValueError):
            sm.setup_dynamic_interp(np.ones((4, 3)), 100)


def test_library_exports_every_declared_symbol():
    _lib.build()
    hdr = open(os.path.join(ROOT, "include", "sonicsim_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    declared = sorted(set(re.findall(r"\b(ss_[a-z_0-9]+)\s*\(", hdr)))
    assert declared, "no declarations parsed"
    lib = ctypes.CDLL(_lib.LIB_PATH)
    for name in declared:
        assert hasattr(lib, name), "library does not export %s" % name
    assert sorted(_lib.EXPORTS) == declared
    assert lib.ss_version() >= 100


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError):
        sm.convolve_fixed_receiver(np.zeros((1, 100), np.float32), np.zeros((1, 10), np.float32))


def test_index_error_like_reference():
    x = np.zeros(10, np.float32)
    h = np.zeros((3, 1, 4), np.float32)
    with pytest.raises(IndexError):
        sm.convolve_moving_receiver(x, h, np.full(10, 2), np.zeros(10, np.float32))   # idx + 1 == P


def test_ctypes_structs_match_the_c_header_layout(tmp_path):
    """The ctypes mirrors in _lib.py against include/sonicsim_b200.h as gcc lays it out: same size and the same
    offset for every field (the header is the contract a maintainer binds against)."""
    import ctypes
    import shutil
    import subprocess
    from sonicsim_b200 import _lib
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    pairs = {"ss_source": _lib.SsSource, "ss_loud_item": _lib.SsLoudItem, "ss_post_lufs": _lib.SsPostLufs,
             "ss_mix_item": _lib.SsMixItem, "ss_dry_clip": _lib.SsDryClip}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sonicsim_b200.h"', 'int main(void) {']
    for cname, cls in pairs.items():
        lines.append('printf("%s size %%zu\\n", sizeof(%s));' % (cname, cname))
        for fname, _ in cls._fields_:
            lines.append('printf("%s %s %%zu\\n", offsetof(%s, %s));' % (cname, fname, cname, fname))
    lines += ['return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    inc = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include")
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", inc, str(src), "-o", str(exe)], check=True)     # the header is plain C
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {tuple(l.split()[:2]): int(l.split()[2]) for l in out if l.strip()}
    for cname, cls in pairs.items():
        assert got[(cname, "size")] == ctypes.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert got[(cname, fname)] == getattr(cls, fname).offset, (cname, fname)


def _plan(N, P, C, L, bounds):
    """ss_debug_plan through ctypes: (blocks (n, 4), aligned)."""
    lib = _lib.load()
    b = np.ascontiguousarray(bounds, dtype=np.int32)
    item = _lib.SsSource(x=1, rir=1, out=1, bounds=b.ctypes.data, N=N, P=P, C=C, L=L, mode=_lib.SS_MOVING_BOUNDS,
                         bounds_host=b.ctypes.data)
    cap = (N + 4095) // 4096 + P
    out = np.zeros((cap, 4), dtype=np.int32)
    aligned = ctypes.c_int32(-1)
    n = lib.ss_debug_plan(ctypes.byref(item), out.ctypes.data, cap, ctypes.byref(aligned))
    assert n >= 0, n
    return out[:n], aligned.value


def test_host_block_planner_invariants_and_choice():
    """The host twin of k_blocks (build_blocks_host / choose_aligned in ss_kernels.cu, pure host code): blocks tile
    [0, N) exactly, never exceed 4096 samples, never cross a waypoint under aligned blocking and carry that segment's
    position pair; the plan chosen is the one with fewer inverse transforms (exact counts from the bounds)."""
    rng = np.random.default_rng(5)
    for case in range(200):
        P = int(rng.integers(2, 70))
        N = int(rng.integers(P, 200000))
        cuts = np.sort(rng.integers(0, N + 1, P - 2)) if rng.random() < 0.8 else np.sort(rng.choice([0, N // 2, N], P - 2))
        bounds = np.concatenate([[0], cuts, [N]]).astype(np.int32)          # zero-length segments allowed
        L = int(rng.choice([1, 300, 4096, 4097, 9000]))
        blocks, aligned = _plan(N, P, 2, L, bounds)
        # exact transform counts of the two plans
        seg = np.diff(bounds.astype(np.int64))
        cost_aligned = int(np.sum((seg + 4095) // 4096))
        cost_grid = 0
        for b0 in range(0, N, 4096):
            n0, n1 = b0, min(b0 + 4096, N) - 1
            lo = int(np.searchsorted(bounds[1:], n0, side="right"))          # segment of the first sample
            hi = int(np.searchsorted(bounds[1:], n1, side="right"))          # ... of the last one
            lo, hi = min(lo, P - 2), min(hi, P - 2)
            cost_grid += (hi - lo + 2 + 1) // 2
        if L > 4096:
            assert aligned == 0                                              # long RIRs stay on the grid
        else:
            assert aligned == (1 if cost_aligned <= cost_grid else 0), (case, cost_aligned, cost_grid)
        # tiling
        order = np.argsort(blocks[:, 0], kind="stable")
        pos = 0
        for s, ln, p_lo, p_hi in blocks[order]:
            assert s == pos and 0 < ln <= 4096
            pos += ln
            if aligned:
                assert p_hi == p_lo + 1 and bounds[p_lo] <= s and s + ln <= bounds[p_lo + 1]
                assert (s - bounds[p_lo]) % 4096 == 0
            else:
                assert s % 4096 == 0
        assert pos == N
        if aligned:
            assert len(blocks) == cost_aligned


def test_chunking_respects_the_budget_and_balances():
    """ss_debug_chunks (pure host): every chunk fits the scratch budget unless a single item is bigger, chunks are
    contiguous and cover the batch, equal items are split into near-equal chunks (ADVICE r1: the budget rule used to be
    measured from an ideal cut position, which let chunks of mixed item sizes grow to twice the budget)."""
    lib = _lib.load()
    rng = np.random.default_rng(0)
    for trial in range(200):
        n = int(rng.integers(1, 60))
        kind = trial % 3
        if kind == 0:
            b = np.full(n, 13 << 20, np.int64)
        elif kind == 1:
            b = rng.integers(1 << 20, 40 << 20, n).astype(np.int64)
        else:
            b = np.where(rng.random(n) < 0.2, 90 << 20, 2 << 20).astype(np.int64)
        budget = int(rng.integers(20 << 20, 120 << 20))
        cuts = np.zeros(n + 1, np.int32)
        k = lib.ss_debug_chunks(b.ctypes.data, n, budget, cuts.ctypes.data, n + 1)
        assert k >= 2
        cuts = cuts[:k]
        assert cuts[0] == 0 and cuts[-1] == n and np.all(np.diff(cuts) > 0)
        sizes = [int(b[a:c].sum()) for a, c in zip(cuts[:-1], cuts[1:])]
        for (a, c), sz in zip(zip(cuts[:-1], cuts[1:]), sizes):
            assert sz <= budget or c - a == 1, (trial, sz, budget)
    # 32 equal items, 7 per budget: 5 chunks of 6-7 items, not 7,7,7,7,4
    b = np.full(32, 13 << 20, np.int64)
    cuts = np.zeros(33, np.int32)
    k = lib.ss_debug_chunks(b.ctypes.data, 32, 96 << 20, cuts.ctypes.data, 33)
    d = np.diff(cuts[:k])
    assert k == 6 and d.min() >= 6 and d.max() <= 7


def test_chunk_budget_fixture_restores_the_library_default():
    """The chunk_budget fixture (tests/chunk_budget.py) puts back the device-path budget a fresh context starts with."""
    from chunk_budget import DEFAULT_CHUNK_BYTES
    src = open(os.path.join(ROOT, "sonicsim_b200", "csrc", "ss_internal.h")).read()
    m = re.search(r"int64_t chunk_bytes = (\d+)ll << (\d+);", src)
    assert m and (int(m.group(1)) << int(m.group(2))) == DEFAULT_CHUNK_BYTES
