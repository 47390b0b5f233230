"""Pair gains (ss_pair_gains; DryPick(..., gains=)) on the CPU: the heads of k_blocks (pick_pooled) and of k_stage
(stage_head), exported by tests/emu/ss_emu_pair.cu, take table[d * n + i] with both picks clamped, in place of the
pool's gain, and a slot without a table keeps the pool's gain; the exports; and the Python refusals that need no
device."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from sonicsim_b200 import _lib


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_pair")


def heads(emu, N, g, tab, n_dry, v, dv):
    Na = np.asarray(N, np.int32)
    ga = np.asarray(g if g is not None else [1.0] * len(N), np.float32)
    ta = np.asarray(tab if tab is not None else [0.0], np.float32)
    out = np.zeros(6)
    emu.emu_pair_heads(Na.ctypes.data, ga.ctypes.data, int(g is not None), len(N), n_dry, ta.ctypes.data,
                       int(tab is not None), v, dv, out.ctypes.data)
    return out


def test_both_heads_take_the_clamped_pairs_gain(emu):
    """With a table, pick_pooled and stage_head store table[d * n + i] (d, i clamped; bits 3 and 4 as without a table)
    whatever the pool's gains; without one, the pool's gain of the clamped candidate (1 for a pool without gains)."""
    rng = np.random.default_rng(11)
    seen = set()
    for n, n_dry in ((1, 1), (3, 5), (7, 2), (13, 11)):
        N = list(rng.integers(5000, 9000, n))
        g = list(rng.uniform(0.1, 4.0, n).astype(np.float32))
        tab = rng.uniform(0.01, 30.0, n * n_dry).astype(np.float32)
        for v in (-(1 << 31), -1, 0, n // 2, n - 1, n, (1 << 31) - 1):
            for dv in (-5, 0, n_dry - 1, n_dry, 1 << 30):
                i, d = min(max(v, 0), n - 1), min(max(dv, 0), n_dry - 1)
                err = (8 if not 0 <= v < n else 0) | (16 if not 0 <= dv < n_dry else 0)
                for pool_gains in (None, g):
                    for table in (tab, None):
                        out = heads(emu, N, pool_gains, table, n_dry, v, dv)
                        if table is not None:
                            want = tab[d * n + i]
                        else:
                            want = pool_gains[i] if pool_gains is not None else np.float32(1.0)
                        assert out[0] == err and out[3] == err, (n, v, dv, out)
                        assert out[2] == d and out[5] == d, (n, v, dv, out)
                        assert np.float32(out[1]) == want and np.float32(out[4]) == want, (n, v, dv, out, want)
                        seen.add(err)
    assert seen == {0, 8, 16, 24}


def test_pair_gains_symbols_are_exported():
    lib = ctypes.CDLL(_lib.build())
    for name in ("ss_pair_gains_create", "ss_pair_gains_bytes", "ss_pair_gains_destroy", "ss_plan_create_pair"):
        assert hasattr(lib, name) and name in _lib.EXPORTS, name
    L = _lib.load()
    assert L.ss_version() == 108
    assert L.ss_pair_gains_bytes(None) == 0
    L.ss_pair_gains_destroy(None)
    h = ctypes.c_void_p()
    t = np.zeros(4)
    assert L.ss_pair_gains_create(None, None, None, None, t.ctypes.data, None, ctypes.byref(h)) == _lib.SS_ERR_INVALID
    assert L.ss_plan_create_pair(None, None, 1, None, 0, None, 0, None, None, 0, ctypes.byref(h)) == \
        _lib.SS_ERR_INVALID
    assert L.ss_plan_create_pair(None, None, 1, None, 0, None, 0, None, None, -1, ctypes.byref(h)) == \
        _lib.SS_ERR_INVALID
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
    other = _FakeRenderer(2000)

    def pool(r=R, **kw):
        a = dict(resident="device", gains=False, _sizes=[3000, 4000], levels=None, n=2, C=2)
        a.update(kw)
        p = _fake(render.SourcePool, r, **a)
        p._h = ctypes.c_void_p(5)
        return p

    def dry(r=R, **kw):
        a = dict(n=3, n_min=5000, levels=False, resident="device")
        a.update(kw)
        d = _fake(render.DryPool, r, **a)
        d._h = ctypes.c_void_p(7)
        return d

    sp, dp = pool(), dry()

    def refuse_build(match, p=sp, d=dp, targets=-20.0, sr=16000):
        with pytest.raises(ValueError, match=match):
            render.Renderer.pair_gains(R, p, d, targets, sr)

    # pair_gains: every check before any C call
    refuse_build("must be a SourcePool", p="pool")
    refuse_build("must be a DryPool", d="dry")
    refuse_build("SourcePool belongs to another renderer", p=pool(other))
    refuse_build("DryPool belongs to another renderer", d=dry(other))
    refuse_build("at most 8 channels", p=pool(C=9))
    refuse_build("shorter than the pool's longest", p=pool(_sizes=[3000, 5001]))
    refuse_build("at most 2\\^26", p=pool(n=1 << 13, _sizes=[3000]), d=dry(n=1 << 14))
    refuse_build("\\(n_dry, n\\) = \\(3, 2\\)", targets=np.zeros((2, 3)))
    refuse_build("\\(n_dry, n\\) = \\(3, 2\\)", targets=[-20.0, -18.0])
    bad = np.full((3, 2), np.nan)
    bad[2, 1] = np.inf
    refuse_build("pair \\(2, 1\\) is not finite", targets=bad)
    refuse_build("is not finite", targets=-np.inf)
    refuse_build("sr must be > 0", sr=0)
    closed = dry()
    closed._closing = True
    refuse_build("DryPool is closed", d=closed)

    # DryPick keeps its two fields; gains is a third, None by default
    a = render.DryPick(dp, "pick")
    assert a.gains is None and a == (dp, "pick", None)

    def gains(p=sp, d=dp, r=R):
        g = _fake(render.PairGains, r, pool=p, dry_pool=d)
        g._h = ctypes.c_void_p(9)
        return g

    def refuse(sources, match):
        with pytest.raises(ValueError, match=match):
            render.Renderer._device_dry(R, sources)

    pk = torch.zeros(1, dtype=torch.int32)
    gp = pool(gains=True)
    refuse([render.Pooled(gp, None, (0, 10), 0, render.DryPick(dp, pk))], "loudness gains")
    refuse([render.Pooled(sp, None, (0, 10), 0, render.DryPick(dp, pk, "g"))], "must be a PairGains")
    refuse([render.Pooled(sp, None, (0, 10), 0, render.DryPick(dp, pk, gains(r=other)))], "another renderer's context")
    g_closed = gains()
    g_closed._closing = True
    refuse([render.Pooled(sp, None, (0, 10), 0, render.DryPick(dp, pk, g_closed))], "PairGains of source 0 is closed")
    refuse([render.Pooled(gp, None, (0, 10), 0, render.DryPick(dp, pk, gains()))], "another SourcePool or DryPool")
    refuse([render.Pooled(sp, None, (0, 10), 0, render.DryPick(dp, pk, gains(d=dry())))], "another SourcePool or DryPool")
    # past the pool checks, on a pool with gains too: the pick tensor (a CPU tensor here) is refused next
    for p in (sp, gp):
        refuse([render.Pooled(p, None, (0, 10), 0, render.DryPick(dp, pk, gains(p=p)))],
               "dry pick of source 0 must be a CUDA tensor")
    # the handle array of ss_plan_create_pair, in the order of the dry picks; None without any gains
    g0 = gains()
    srcs = [render.Pooled(sp, None, (0, 10), 0, render.DryPick(dp, pk)), render.Pooled(sp, None, (0, 10)),
            render.Pooled(sp, None, (0, 10), 0, render.DryPick(dp, pk, g0))]
    arr = render.Renderer._device_pair_gains(srcs)
    assert [arr[0], arr[1]] == [None, 9] and len(arr) == 2
    assert render.Renderer._device_pair_gains(srcs[:2]) is None
    for o in (sp, dp, g0, g_closed):
        o._h = ctypes.c_void_p(0)
