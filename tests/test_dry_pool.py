"""Dry pools (ss_dry_pool; dry-picked pooled slots, ss_dry_pick) on the CPU: the head of k_blocks on a dry-picked slot
(pick_pooled of ss_phases.cuh, exported by tests/emu/ss_emu_dry_pool.cu) - the clamps, the error bits, x replaced while
everything else comes from the trajectory candidate; k_draw's choice of each speaker's table (speaker_table) in draws
that mix dry-picked speakers and pooled ones, against tests/draw_reference.py; the ctypes mirror of ss_dry_pick against
gcc; the exports; and the refusals that need no device."""
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


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_dry_pool")


def pick(emu, N, P, Ks=None, gains=None, K=1, C=2, direct=0, n_dry=0, v=0, dv=0):
    Na, Pa = np.asarray(N, np.int32), np.asarray(P, np.int32)
    Ka = np.asarray(Ks if Ks is not None else [K] * len(N), np.int32)
    ga = np.asarray(gains if gains is not None else [1.0] * len(N), np.float32)
    out = np.zeros(11)
    emu.emu_pick_pooled(Na.ctypes.data, Pa.ctypes.data, Ka.ctypes.data, int(Ks is not None), ga.ctypes.data,
                        int(gains is not None), len(N), K, C, direct, n_dry, v, dv, out.ctypes.data)
    return dict(err=int(out[0]), x=int(out[1]), N=int(out[2]), P=int(out[3]), K=int(out[4]), nb=int(out[5]),
                bounds=int(out[6]), spec=int(out[7]), cut=int(out[8]), h_rows=int(out[9]), gain=float(out[10]))


def test_head_without_a_dry_pick_keeps_the_candidates_x(emu):
    N, P = [30000, 41000, 9000], [3, 5, 2]
    for v, want, err in [(1, 1, 0), (7, 2, 8), (-4, 0, 8)]:
        r = pick(emu, N, P, n_dry=0, v=v, dv=99)
        assert r["x"] == -1 - want and r["err"] == err, (v, r)
        assert (r["N"], r["P"], r["bounds"], r["spec"]) == (N[want], P[want], want, want)


def test_head_replaces_x_only(emu):
    """x is the dry pool's signal dry_pick names (clamped, bit 4); N, P, nb, bounds, K, spectra, cuts, h_rows and gain are
    the picked trajectory candidate's, with mixed K and gains, with and without a direct stem."""
    N, P, Ks, g = [30000, 41000, 9000, 5000], [3, 5, 2, 1 + 1], [1, 3, 2, 1], [0.5, 2.0, 1.25, 3.0]
    seen = set()
    for v in (-1, 0, 1, 2, 3, 4, 1 << 30):
        for dv in (-(1 << 31), -1, 0, 5, 6, 7, (1 << 31) - 1):
            for direct in (0, 1):
                for parts, gains in ((Ks, g), (None, None)):
                    n_dry = 7
                    r = pick(emu, N, P, Ks=parts, gains=gains, K=3, C=2, direct=direct, n_dry=n_dry, v=v, dv=dv)
                    c = min(max(v, 0), len(N) - 1)
                    d = min(max(dv, 0), n_dry - 1)
                    err = (8 if not 0 <= v < len(N) else 0) | (16 if not 0 <= dv < n_dry else 0)
                    K = Ks[c] if parts else 3
                    assert r["err"] == err and r["x"] == d, (v, dv, r)
                    assert (r["N"], r["P"], r["nb"], r["K"]) == (N[c], P[c], (N[c] + 4095) // 4096, K), (v, dv, r)
                    assert (r["bounds"], r["spec"], r["cut"]) == (c, c, c if direct else -1)
                    assert r["h_rows"] == P[c] * 2 * K
                    assert r["gain"] == (np.float32(g[c]) if gains else 1.0)
                    seen.add(err)
    assert seen == {0, 8, 16, 24}


def _gappy(rng, N):
    y = (0.05 * rng.standard_normal(N)).astype(np.float32)
    pos = 0
    while pos < N:
        gap = int(rng.integers(0, N // 3))
        y[pos:pos + gap] = 0
        pos += gap + int(rng.integers(N // 10, N // 3))
    return y


def test_draws_with_dry_and_pooled_speakers(emu):
    """Readers of pools of different N; speakers with a dry pick (one-channel dry tables, D = len) and without (pool
    tables, mono or C channels) in one draw; picks and dry picks out of range (clamped); passing, later and all-silent
    draws.  The emulated draw equals draw_reference on the tables the picks name; M comes from the trajectory picks."""
    rng = np.random.default_rng(21)
    seen = set()
    for case in range(200):
        length = int(rng.integers(40, 300))
        n_readers = int(rng.integers(1, 6))
        S = int(rng.integers(1, n_readers + 1))
        C = int(rng.integers(1, 4))
        mono = bool(case % 2)
        cand_N, cand_Q, cand_off, cand_n = [], [], [], []
        dry_Q, dry_off, dry_n, dry_tabs = [], [], [], []
        picks, dry_picks = [], []
        for r in range(n_readers):
            n = int(rng.integers(1, 4))
            cand_off.append(len(cand_N))
            cand_n.append(n)
            for _ in range(n):
                N = int(rng.integers(length, 10 * length))
                cand_N.append(N)
                y = np.stack([_gappy(rng, N) for _ in range(C)])
                cand_Q.append(dr.level_table(y, mono))
            nd = int(rng.integers(1, 4)) if rng.random() < 0.5 else 0
            dry_off.append(len(dry_Q))
            dry_n.append(nd)
            tabs = []
            for _ in range(nd):
                # dry signals at least as long as every candidate of the reader's pool
                x = _gappy(rng, max(cand_N[cand_off[r]:cand_off[r] + n]) + int(rng.integers(0, 50)))
                dry_Q.append(dr.level_table(x[None], True))
                tabs.append(dry_Q[-1])
            dry_tabs.append(tabs)
            picks.append(int(rng.integers(-1, n + 1)))
            dry_picks.append(int(rng.integers(-1, nd + 1)))
        spk = list(rng.permutation(n_readers)[:S])
        D = [length * (1 if mono else C)] * S
        tries = int(rng.integers(1, 60))
        u = rng.random(tries)
        thr = 100.0 if case % 7 == 0 else -40.0 if case % 3 else -25.0
        clamp = lambda v, n: min(max(v, 0), n - 1)                          # noqa: E731
        reader_N = [cand_N[cand_off[r] + clamp(picks[r], cand_n[r])] for r in range(n_readers)]
        tabs, Ds = [], []
        for k, r in enumerate(spk):
            if dry_n[r]:
                tabs.append(dry_tabs[r][clamp(dry_picks[r], dry_n[r])])
                Ds.append(length)
            else:
                tabs.append(cand_Q[cand_off[r] + clamp(picks[r], cand_n[r])])
                Ds.append(D[k])
        want = dr.draw(tabs, Ds, reader_N, length, u, thr)
        if dr.margins(tabs, Ds, reader_N, length, u, thr) < 1e-9:
            continue
        i32 = lambda a: np.ascontiguousarray(a, np.int32)                   # noqa: E731
        cq = (ctypes.c_void_p * len(cand_Q))(*[q.ctypes.data for q in cand_Q])
        dq = (ctypes.c_void_p * max(1, len(dry_Q)))(*[q.ctypes.data for q in dry_Q])
        arrs = [i32(cand_N), i32(cand_off), i32(cand_n), i32(picks), i32(dry_off), i32(dry_n), i32(dry_picks),
                i32(spk), np.ascontiguousarray(D, np.float64), np.ascontiguousarray(u, np.float64)]
        cN, co, cn, pk, do, dn, dp, sp, Da, ua = arrs
        used = ctypes.c_int32()
        s = emu.emu_draw_mixed(cN.ctypes.data, ctypes.cast(cq, ctypes.c_void_p), co.ctypes.data, cn.ctypes.data,
                               pk.ctypes.data, ctypes.cast(dq, ctypes.c_void_p), do.ctypes.data, dn.ctypes.data,
                               dp.ctypes.data, n_readers, sp.ctypes.data, Da.ctypes.data, S, length, ua.ctypes.data,
                               tries, thr, ctypes.byref(used))
        assert (s, used.value) == want, case
        kinds = {bool(dry_n[r]) for r in spk}
        seen.add(("mixed" if kinds == {True, False} else "dry" if kinds == {True} else "pool") +
                 ("-none" if want[1] == 0 else "-first" if want[1] == 1 else "-later"))
    assert {"mixed-first", "mixed-later", "mixed-none", "dry-first", "dry-none", "pool-first"} <= seen, seen


def test_ss_dry_pick_layout(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "sonicsim_b200.h"', 'int main(void) {',
             'printf("size %zu\\n", sizeof(ss_dry_pick));']
    for fname, _ in _lib.SsDryPick._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(ss_dry_pick, %s));' % (fname, fname))
    lines += ['printf("levels %u\\n", SS_DRY_LEVELS);', 'return 0;', '}']
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                    str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {l.split()[0]: int(l.split()[1]) for l in out if l.strip()}
    assert got["size"] == ctypes.sizeof(_lib.SsDryPick)
    for fname, _ in _lib.SsDryPick._fields_:
        assert got[fname] == getattr(_lib.SsDryPick, fname).offset, fname
    assert got["levels"] == _lib.SS_DRY_LEVELS


def test_dry_pool_symbols_are_exported():
    lib = ctypes.CDLL(_lib.build())
    for name in ("ss_dry_pool_create", "ss_dry_pool_bytes", "ss_dry_pool_level_table", "ss_dry_pool_destroy",
                 "ss_plan_create_dry"):
        assert hasattr(lib, name) and name in _lib.EXPORTS, name
    L = _lib.load()
    assert L.ss_version() == 108
    assert L.ss_dry_pool_bytes(None) == 0
    assert L.ss_dry_pool_level_table(None, 0) is None
    L.ss_dry_pool_destroy(None)
    h = ctypes.c_void_p()
    x = (ctypes.c_void_p * 1)(4096)
    n = np.array([100], np.int32)
    assert L.ss_dry_pool_create(None, x, n.ctypes.data, 1, 0, ctypes.byref(h)) == _lib.SS_ERR_INVALID
    assert L.ss_plan_create_dry(None, None, 1, None, 0, None, 0, None, 0, ctypes.byref(h)) == _lib.SS_ERR_INVALID
    assert L.ss_plan_create_dry(None, None, 1, None, 0, None, 0, None, -1, ctypes.byref(h)) == _lib.SS_ERR_INVALID
    assert not h.value


class _FakeRenderer:
    def __init__(self, ctx):
        self.ctx, self.device = ctypes.c_void_p(ctx), 0


def _fake(cls, renderer, **kw):
    obj = object.__new__(cls)
    obj.renderer, obj._h = renderer, ctypes.c_void_p(0)      # a null handle: nothing to free
    for k, v in kw.items():
        setattr(obj, k, v)
    return obj


def test_python_refusals_without_a_device():
    from sonicsim_b200 import render
    torch = pytest.importorskip("torch")
    R = _FakeRenderer(1000)
    # dry_pool: counts and tensors are checked before any C call
    with pytest.raises(ValueError, match="1 to 2\\^24 signals"):
        render.Renderer.dry_pool(R, [])
    with pytest.raises(ValueError, match="CUDA tensor"):
        render.Renderer.dry_pool(R, [torch.zeros(10)])

    dp = _fake(render.DryPool, R, n=3, n_min=5000, levels=False)
    dp._h = ctypes.c_void_p(7)

    def pool(**kw):
        a = dict(resident="device", gains=False, _sizes=[3000, 4000], levels=None)
        a.update(kw)
        return _fake(render.SourcePool, R, **a)

    def refuse(sources, match):
        with pytest.raises(ValueError, match=match):
            render.Renderer._device_dry(R, sources)

    dpick = render.DryPick(dp, torch.zeros(1, dtype=torch.int32))
    # a DryPick on a source that is not pooled
    refuse([render.MovingSource(dpick, None, None)], "not a pooled slot")
    refuse([render.Pooled(pool(), None, (0, 10), 0, "x")], "DryPick or None")
    refuse([render.Pooled(pool(), None, (0, 10), 0, render.DryPick(object(), None))], "must be a DryPool")
    refuse([render.Pooled(pool(resident="host"), None, (0, 10), 0, dpick)], "host pool")
    refuse([render.Pooled(pool(gains=True), None, (0, 10), 0, dpick)], "loudness gains")
    refuse([render.Pooled(pool(_sizes=[3000, 5001]), None, (0, 10), 0, dpick)], "shorter than its pool's longest")
    # the pick tensor: checked after the pools (a CPU tensor here)
    refuse([render.Pooled(pool(), None, (0, 10), 0, dpick)], "dry pick of source 0 must be a CUDA tensor")
    other = _fake(render.DryPool, _FakeRenderer(2000), n=3, n_min=5000, levels=False)
    other._h = ctypes.c_void_p(8)
    refuse([render.Pooled(pool(), None, (0, 10), 0, render.DryPick(other, dpick.pick))], "another renderer's context")
    dp._closing = True
    refuse([render.Pooled(pool(), None, (0, 10), 0, dpick)], "is closed")
    dp._closing = False
    # no dry picks: nothing to pass
    assert render.Renderer._device_dry(R, [render.Pooled(pool(), None, (0, 10))]) is None
    dp._h = other._h = ctypes.c_void_p(0)


def test_pooled_keeps_its_fields():
    from sonicsim_b200 import render
    a = render.Pooled("pool", "pick", (0, 10))
    assert a.direct_taps == 0 and a.dry is None
    assert render.Pooled("pool", "pick", (0, 10), 40) == ("pool", "pick", (0, 10), 40, None)
