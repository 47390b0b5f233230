"""The host path (ss_render_host_ex) at bench scale against float64.  It copies each chunk's read sets into one of four
device slots (chunk k on slot k % 4, reused once the slot's copies out are done), renders on one stream, measures and
normalises loudness on side stream k % 3 in place in the slot, and copies stems and loudness results back; its slots,
its loudness block (h_post / d_post) and the first slot's scratch for the stand-alone host entries grow on demand.  A
stem copied from the wrong span, a result written to the wrong stem or a slot reused too early gives plausible audio,
so every stem here is checked sample by sample against the float64 render reference (render_reference.check_render,
direct stems against direct_path_rirs, normalised RIRs against direct_path.normalized), every loudness result against
the float64 BS.1770 oracle on the device's own raw stem, and every host output sits in a NaN-filled buffer with
sentinels on both sides, pinned where bench.py pins and pageable elsewhere.
  A. bench.py's end-to-end batch (32 configs[1] speakers), plan_host run twice with new dry signals in the bound pinned
     buffers, then once more over pageable buffers: more than 2 x kSlots chunks;
  B. scene_lufs at that scale: a different target per stem, some None, direct stems; and the all -17 LUFS batch as
     bench.py builds it, which puts loudness work on every side stream;
  C. one heterogeneous batch (bounds, indexed, static, long-RIR, banked, normalised, direct, windowed, loudness) on
     contexts with 1 MB, the default and 512 MB host budgets, the last one holding every source in one slot;
  D. growth: a sequence of calls on a fresh context whose slots, loudness block and scratch reallocate between and
     within calls, and the stand-alone host entries (ss_lufs_norm_host, ss_mix_host_ex, ss_overlap_host) through
     rising and falling sizes;
  E. the drop-in (SonicSim_moving) at full configs[1] size.
The float64 references of the bench sources are computed once for the module (render_check_inputs piecewise, with
enough context around every piece that the result is the whole stem's)."""
import contextlib
import ctypes
import os
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import bench
from direct_path import direct_path_rirs, normalized
from mix_reference import F32, overlap_exact
from oracle import sonicsim_oracle as so
from render_reference import F, TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from window_cases import _host_aligned, poison, read_set
from gpu_plumbing import _R, _workers, pmap
from loudness_cases import EXACT_DB, assert_clear_of_gates, block_size_of
from mix_reference import check_mix

pytestmark = pytest.mark.gpu

RATE = 16000
SENT = np.float32(1234.5)
PAD = 37
TAPS = 40
K_SLOTS = 4                      # ss_ctx::kSlots
K_AUX = 3                        # ss_ctx::kAux
LOUD_SCRATCH_DOUBLES = 20        # SS_LOUD_SCRATCH_DOUBLES
MB = 1 << 20
STATS = {}                       # section -> [worst local ratio, worst global relative RMS]
LUFS = {}                        # section -> worst |LUFS - float64 oracle|


def _note(key, worst, g):
    s = STATS.setdefault(key, [0.0, 0.0])
    s[0], s[1] = max(s[0], worst), max(s[1], g)


def _report(section):
    for k in sorted(STATS):
        if k.startswith(section):
            print("\n%-28s worst per-sample ratio %.3g (bound %.3g), worst global relative RMS %.3g (bound %.3g)"
                  % (k, STATS[k][0], TAU_LOCAL, STATS[k][1], TAU_GLOBAL), end="")
    for k in sorted(LUFS):
        if k.startswith(section):
            print("\n%-28s worst |LUFS - float64| %.3g dB" % (k, LUFS[k]), end="")
    print()


# ------------------------------------------------------------------------------------------------ references
def reference(x, h, mode, bounds=None, idx=None, w=None, window=None, piece=1 << 16):
    """render_check_inputs of output samples [a, a + n) (window (a, n), default the whole stem), computed piece by
    piece: each piece with F samples of context on both sides inside [a, a + n), which is all its peak filter reads,
    and the 2^-30 max |y64| term taken over the whole range, so that the result is the one-piece result.  A moving
    source convolves only the positions a piece visits, not all P of them over the whole stem."""
    N = len(x)
    a, n = (0, N) if window is None else (int(window[0]), int(window[1]))
    ys, ss = [], []
    for p0 in range(a, a + n, piece):
        p1 = min(a + n, p0 + piece)
        c0, c1 = max(a, p0 - F), min(a + n, p1 + F)
        y, s = render_check_inputs(x, h, mode, bounds, idx, w, window=(c0, c1 - c0))
        ys.append(y[:, p0 - c0:p1 - c0])
        ss.append(s[:, p0 - c0:p1 - c0] - np.abs(y).max() * 2.0 ** -30)
    y = np.concatenate(ys, axis=1)
    s = np.concatenate(ss, axis=1) + np.abs(y).max() * 2.0 ** -30
    return y, s.astype(np.float32)


def check(key, y, ref, n0=0, label="", gain=None):
    """check_render of stem y against ref = (y64, scale), both scaled by float32(gain) when given."""
    y64, scale = ref
    if gain is not None:
        g = float(np.float32(gain))
        y64, scale = y64 * g, scale.astype(np.float64) * g
    worst, gl = check_render(y, y64, scale.astype(np.float64), TAU_LOCAL, TAU_GLOBAL, n0=n0, label=label)
    return key, worst, gl


def _noted(results):
    for key, worst, gl in results:
        _note(key, worst, gl)


def check_loudness(key, raw, out, lufs, gain, target, label, raw_d=None, out_d=None):
    """LUFS of the (C, N) raw stem against the float64 BS.1770 oracle within EXACT_DB, gain == 10^((t - LUFS) / 20),
    out == float32(gain) * raw bit for bit, and the direct stem scaled by the same gain."""
    stem = np.ascontiguousarray(raw.T)
    assert_clear_of_gates(stem, RATE, block_size_of(stem.shape[0], RATE))
    ref = so.bs1770_integrated_loudness(stem, RATE, block_size_of(stem.shape[0], RATE), up_to_8_channels=True)
    assert abs(lufs - ref) <= EXACT_DB, (label, lufs, ref)
    assert gain == pytest.approx(10 ** ((target - lufs) / 20), rel=1e-13), label
    assert np.array_equal(out, np.float32(gain) * raw), label
    if raw_d is not None:
        assert np.array_equal(out_d, np.float32(gain) * raw_d), label
    LUFS[key] = max(LUFS.get(key, 0.0), abs(lufs - ref))


class Out:
    """A (C, n) float32 host output inside a NaN-filled buffer with PAD sentinels on both sides, pinned or pageable."""

    def __init__(self, C, n, pinned):
        size = C * n + 2 * PAD
        self.t = torch.empty(size, dtype=torch.float32).pin_memory() if pinned else None
        self.buf = self.t.numpy() if pinned else np.empty(size, np.float32)
        self.C, self.n = C, n
        self.reset()

    def reset(self):
        self.buf[:PAD] = SENT
        self.buf[-PAD:] = SENT
        self.buf[PAD:-PAD] = np.nan

    def view(self):
        return self.buf[PAD:-PAD].reshape(self.C, self.n)

    def get(self, label=""):
        assert np.all(self.buf[:PAD] == SENT) and np.all(self.buf[-PAD:] == SENT), "%s: sentinel overwritten" % label
        v = self.view()
        assert not np.isnan(v).any(), "%s: output samples never written" % label
        return v


class Guard:
    """A 1-D host array of `data` (or n NaNs) between NaN guards of PAD elements; the guards must stay NaN."""

    def __init__(self, data=None, n=None, dtype=np.float32):
        data = None if data is None else np.ascontiguousarray(data, dtype).reshape(-1)
        self.n = data.size if data is not None else int(n)
        self.buf = np.full(self.n + 2 * PAD, np.nan, dtype)
        if data is not None:
            self.buf[PAD:PAD + self.n] = data

    @property
    def ptr(self):
        return self.buf.ctypes.data + PAD * self.buf.itemsize

    def get(self):
        assert np.all(np.isnan(self.buf[:PAD])) and np.all(np.isnan(self.buf[PAD + self.n:])), "guard overwritten"
        return self.buf[PAD:PAD + self.n]


@contextlib.contextmanager
def host_budget_renderer(mb):
    """A Renderer over a context of its own whose host pipeline budget is `mb` MB (SS_HOST_CHUNK_MB is read by
    ss_create; None: the default budget), destroyed on exit.  Its banks and plans belong to that context."""
    render, R = _R()
    old = os.environ.get("SS_HOST_CHUNK_MB")
    if mb is None:
        os.environ.pop("SS_HOST_CHUNK_MB", None)
    else:
        os.environ["SS_HOST_CHUNK_MB"] = str(mb)
    ctx = ctypes.c_void_p()
    try:
        assert R.lib.ss_create(R.device, ctypes.byref(ctx)) == 0
    finally:
        if old is None:
            os.environ.pop("SS_HOST_CHUNK_MB", None)
        else:
            os.environ["SS_HOST_CHUNK_MB"] = old
    Rc = render.Renderer.__new__(render.Renderer)
    Rc.lib, Rc.device, Rc.ctx = R.lib, R.device, ctx
    try:
        yield Rc
    finally:
        torch.cuda.synchronize()
        R.lib.ss_destroy(ctx)


# ------------------------------------------------------------------------------------------------ bench batch
@pytest.fixture(scope="module")
def bench_items():
    return bench.make_inputs(16, 0)                      # 32 configs[1] speakers, as bench.py's rank 0


@pytest.fixture(scope="module")
def bench_refs(bench_items):
    t0 = time.time()
    refs = pmap(lambda it: reference(it[0], it[1], 1, bounds=it[2]), bench_items)
    print("\nfloat64 references of the %d bench stems: %.1f s on %d threads" % (len(refs), time.time() - t0,
                                                                                 _workers()))
    return refs


@pytest.fixture(scope="module")
def bench_pinned(bench_items):
    """The bench batch's inputs pinned as bench.py's run_ours pins them, and its MovingSources over them."""
    render, _ = _R()
    h_items = [(torch.from_numpy(x).pin_memory(), torch.from_numpy(h).pin_memory(), b) for x, h, b in bench_items]
    srcs = [render.MovingSource(x.numpy(), h.numpy(), b) for x, h, b in h_items]
    return SimpleNamespace(items=h_items, srcs=srcs)


def _chunks_of(launches):
    """Chunks of a host call over the bench batch without loudness: k_prepare and k_render per chunk (bounds on the
    host: no k_blocks)."""
    assert launches % 2 == 0, launches
    return launches // 2


def test_a_bench_end_to_end_batch(bench_items, bench_refs, bench_pinned):
    render, R = _R()
    C, N = bench.CFG["C"], bench.CFG["N"]
    n = len(bench_items)
    outs = [Out(C, N, True) for _ in range(n)]
    plan = R.plan_host(bench_pinned.srcs, [o.view() for o in outs])
    c0 = R.launch_count()
    plan.run()
    chunks = _chunks_of(R.launch_count() - c0)
    print("\nA: %d sources in %d chunks" % (n, chunks))
    assert chunks > 2 * K_SLOTS                 # every slot reused at least once within the call
    _noted(pmap(lambda i: check("A run 1", outs[i].get("A %d" % i), bench_refs[i], label="A run 1 stem %d" % i),
                range(n)))
    # new dry contents written into the bound pinned buffers: the same plan renders them
    rng = np.random.default_rng(7331)
    new = [so.synth_dry(rng, N) for _ in range(n)]
    for (hx, _, _), x2 in zip(bench_pinned.items, new):
        hx.numpy()[:] = x2
    for o in outs:
        o.reset()
    c0 = R.launch_count()
    plan.run()
    assert _chunks_of(R.launch_count() - c0) == chunks

    def second(i):
        _, h, b = bench_items[i]
        return check("A run 2", outs[i].get("A2 %d" % i), reference(new[i], h, 1, bounds=b), label="A run 2 stem %d" % i)
    _noted(pmap(second, range(n)))
    for (hx, _, _), (x, _, _) in zip(bench_pinned.items, bench_items):
        hx.numpy()[:] = x
    # pageable inputs and outputs on every other stem, the first run's references again
    srcs = [s if i % 2 == 0 else render.MovingSource(np.array(x), np.array(h), b)
            for i, (s, (x, h, b)) in enumerate(zip(bench_pinned.srcs, bench_items))]
    outs3 = [Out(C, N, i % 2 == 0) for i in range(n)]
    R.plan_host(srcs, [o.view() for o in outs3]).run()
    _noted(pmap(lambda i: check("A pageable", outs3[i].get("A3 %d" % i), bench_refs[i], label="A pageable stem %d" % i),
                range(n)))
    _report("A")


B_DIRECT = (2, 9, 16, 31)        # stems with direct targets
B_NONE = (5, 14, 23)             # stems without a loudness target


def test_b_scene_lufs_at_scale(bench_items, bench_refs, bench_pinned):
    render, R = _R()
    C, N = bench.CFG["C"], bench.CFG["N"]
    n = len(bench_items)
    srcs = [s._replace(direct_taps=TAPS) if i in B_DIRECT else s for i, s in enumerate(bench_pinned.srcs)]
    targets = [None if i in B_NONE else -13.0 - 0.61 * i for i in range(n)]
    # raw stems: pinned reverberant outputs, pageable direct outputs
    raw = [Out(C, N, True) for _ in range(n)]
    raw_d = {i: Out(C, N, False) for i in B_DIRECT}
    R.plan_host(srcs, [o.view() for o in raw], direct_outs=[raw_d[i].view() if i in raw_d else None
                                                             for i in range(n)]).run()
    raw = [o.get("B raw %d" % i) for i, o in enumerate(raw)]
    raw_d = {i: o.get("B raw direct %d" % i) for i, o in raw_d.items()}
    _noted(pmap(lambda i: check("B raw", raw[i], bench_refs[i], label="B raw stem %d" % i), range(n)))
    _noted(pmap(lambda i: check("B raw direct", raw_d[i], reference(
        bench_items[i][0], direct_path_rirs(bench_items[i][1], TAPS), 1, bounds=bench_items[i][2]),
        label="B raw direct stem %d" % i), B_DIRECT))
    # a different target per stem: pageable reverberant outputs on odd stems, pinned direct outputs
    outs = [Out(C, N, i % 2 == 0) for i in range(n)]
    dd = {i: Out(C, N, True) for i in B_DIRECT}
    plan = R.plan_host(srcs, [o.view() for o in outs], targets, RATE,
                       direct_outs=[dd[i].view() if i in dd else None for i in range(n)])
    plan.run()
    loud = plan.loudness()

    def one(i):
        out = outs[i].get("B %d" % i)
        if targets[i] is None:
            assert np.array_equal(out, raw[i]) and all(np.isnan(loud[i])), i
            if i in dd:
                assert np.array_equal(dd[i].get(), raw_d[i])
            return
        check_loudness("B per-stem targets", raw[i], out, loud[i][0], loud[i][1], targets[i], "B stem %d" % i,
                       raw_d.get(i), dd[i].get("B direct %d" % i) if i in dd else None)
    pmap(one, range(n))
    # bench.py's scene_lufs batch: every stem at -17 LUFS over the pinned buffers, so every chunk (more than kAux of
    # them, see A) runs loudness work on its side stream k % kAux
    h_outs = [Out(C, N, True) for _ in range(n)]
    c0 = R.launch_count()
    R.plan_host(bench_pinned.srcs, [o.view() for o in h_outs]).run()
    chunks = _chunks_of(R.launch_count() - c0)
    assert chunks > 2 * K_SLOTS and chunks >= K_AUX
    for o in h_outs:
        o.reset()
    plan_l = R.plan_host(bench_pinned.srcs, [o.view() for o in h_outs], lufs_targets=[-17.0] * n, sr=RATE)
    plan_l.run()
    loud = plan_l.loudness()
    pmap(lambda i: check_loudness("B all -17", raw[i], h_outs[i].get("B -17 %d" % i), loud[i][0], loud[i][1], -17.0,
                                  "B -17 stem %d" % i), range(n))
    _report("B")


# ------------------------------------------------------------------------------------------------ C. every array kind
class Hetero:
    """One heterogeneous batch for renderer Rc: Python-API sources (bounds, static, long RIRs, a RirBank of Rc's
    context, normalised RIRs, direct targets, windows) plus SS_MOVING_INDEXED sources appended through the C ABI.
    Windowed sources read their own copies of the inputs, NaN (idx: out of range) outside the documented read set."""

    def __init__(self, Rc, rng):
        render, _ = _R()
        from sonicsim_b200 import _lib
        self.specs = []      # (label, mode, x, h_eff (P, C, L) for the reference, bounds, idx, w, window, direct h)

        def moving(P, C, L, N):
            x = so.synth_dry(rng, N)
            h = so.synth_rirs(rng, P, C, L)
            np.random.seed(int(rng.integers(1 << 30)))
            idx, _ = so.setup_dynamic_interp(so.synth_path(rng, P), N)
            b = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)
            return x, h, b

        srcs, targets, self.keep = [], [], []
        mv = moving(8, 2, 2000, 100003)                     # whole moving source with a direct stem
        mn = moving(5, 3, 4096, 81234)
        mn = (mn[0], mn[1] * np.float32(3.7), mn[2])       # raw RIRs: normalised on the device
        st = (so.synth_dry(rng, 77777), so.synth_rirs(rng, 1, 5, 3000), None)
        lg = moving(4, 2, 9000, 60001)                      # two RIR partitions
        ls = (so.synth_dry(rng, 50000), so.synth_rirs(rng, 1, 1, 16384))   # four
        bk = moving(6, 2, 4096, 90001)
        self.bank = Rc.rir_bank(bk[1], direct_taps=TAPS)

        def add(label, s, x, h, bounds, window, target, direct):
            mode = 0 if bounds is None else 1
            srcs.append(s)
            targets.append(target)
            self.specs.append((label, mode, x, h, bounds, None, None, window, direct))

        def windowed(x, h, b, win, normalize=False, banked=False):
            mode = 0 if b is None else 1
            P, C, L = h.shape
            al = _host_aligned(mode, P, C, L, len(x), b)
            rs = read_set(mode, P, C, L, len(x), b, al, win, normalize, True)
            x2, h2, _, _ = poison(x, h, None, None, rs)
            return x2, (None if banked else h2)

        add("bounds+direct", render.MovingSource(mv[0], mv[1], mv[2], direct_taps=TAPS), mv[0], mv[1], mv[2], None,
            -21.0, True)
        add("normalize", render.MovingSource(mn[0], mn[1], mn[2], normalize_rirs=True), mn[0], normalized(mn[1]),
            mn[2], None, -26.0, False)
        add("static", render.StaticSource(st[0], st[1][0]), st[0], st[1], None, None, -19.0, False)
        add("long 9000", render.MovingSource(*lg), lg[0], lg[1], lg[2], None, None, False)
        add("long 16384", render.StaticSource(ls[0], ls[1][0]), ls[0], ls[1], None, None, -30.0, False)
        add("banked+direct", render.MovingSource(bk[0], self.bank, bk[2], direct_taps=TAPS), bk[0], bk[1], bk[2],
            None, -24.0, True)
        for label, (x, h, b), win, direct, banked in (
                ("banked window %4 = 1", bk, (12345, 30000), False, True),
                ("window at 0", mv, (0, 20000), False, False),
                ("window at N - len +direct", mv, (100003 - 17001, 17001), True, False),
                ("long window", lg, (4099, 9000), False, False),
                ("static window < block", st, (40001, 1000), False, False),
                ("normalize window %4 = 2", mn, (30002, 25000), False, False)):
            norm = label.startswith("normalize")
            hr = mn[1] if norm else h
            x2, h2 = windowed(x, hr, b, win, norm, banked)
            if b is None:
                s = render.StaticSource(x2, h2[0], window=win)
            else:
                s = render.MovingSource(x2, self.bank if banked else h2, b, normalize_rirs=norm,
                                        direct_taps=TAPS if direct else 0, window=win)
            add(label, s, x, normalized(hr) if norm else h, b, win, None, direct)
        self.srcs, self.targets = srcs, targets
        # indexed sources (C ABI): whole, and a window whose idx / w are out of range / NaN outside the read set
        P, C, L, N = 6, 3, 600, 50001
        x = so.synth_dry(rng, N)
        h = so.synth_rirs(rng, P, C, L)
        np.random.seed(4)
        idx, w = so.setup_dynamic_interp(so.synth_path(rng, P), N)
        idx = idx.astype(np.int32)
        self.indexed = []
        for label, win in (("indexed", None), ("indexed window", (7001, 15000))):
            if win is None:
                xs, hs, ids, ws = x, h, idx, w
            else:
                xs, hs, ids, ws = poison(x, h, idx, w, read_set(2, P, C, L, N, None, 0, win))
            arrs = [np.ascontiguousarray(a) for a in (xs, hs, ids, ws)]
            self.keep.append(arrs)
            it = _lib.SsSource(x=arrs[0].ctypes.data, rir=arrs[1].ctypes.data, idx=arrs[2].ctypes.data,
                               w=arrs[3].ctypes.data, N=N, P=P, C=C, L=L, mode=_lib.SS_MOVING_INDEXED)
            if win is not None:
                it.win_start, it.win_len = win
            self.indexed.append(it)
            self.specs.append((label, 2, x, h, None, idx, w, win, False))

    def out_shape(self, k):
        label, mode, x, h, b, idx, w, win, direct = self.specs[k]
        return h.shape[1], len(x) if win is None else win[1]

    def run(self, Rc, lufs, pinned):
        """Render the batch once (with the loudness targets when `lufs`); returns (stems, direct stems, loudness,
        launches)."""
        from sonicsim_b200 import _lib
        n_py = len(self.srcs)
        outs = [Out(*self.out_shape(k), pinned=(k % 2 == 0) == pinned) for k in range(len(self.specs))]
        dd = [Out(*self.out_shape(k), pinned=not pinned) if self.specs[k][8] else None for k in range(n_py)]
        plan = Rc.plan_host(self.srcs, [o.view() for o in outs[:n_py]], self.targets if lufs else None, RATE,
                            direct_outs=[d.view() if d is not None else None for d in dd])
        extra = []
        for o, it in zip(outs[n_py:], self.indexed):
            e = _lib.SsSource.from_buffer_copy(it)
            e.out = o.view().ctypes.data
            extra.append(e)
        n = n_py + len(extra)
        items = (_lib.SsSource * n)(*list(plan.items), *extra)
        post = (_lib.SsPostLufs * n)(*list(plan.post), *[_lib.SsPostLufs() for _ in extra]) if lufs else None
        c0 = Rc.launch_count()
        _lib.check(Rc.lib.ss_render_host_ex(Rc.ctx, items, n, post))
        launches = Rc.launch_count() - c0
        stems = [o.get("C %s" % s[0]) for o, s in zip(outs, self.specs)]
        dstems = [d.get("C direct %s" % s[0]) if d is not None else None for d, s in zip(dd, self.specs)]
        loud = plan.loudness() if lufs else None
        return stems, dstems, loud, launches

    def references(self):
        def one(k):
            label, mode, x, h, b, idx, w, win, direct = self.specs[k]
            hh = h if mode else h[0]
            ref = reference(x, hh, mode, bounds=b, idx=idx, w=w, window=win)
            dref = None
            if direct:
                hd = direct_path_rirs(h, TAPS)
                dref = reference(x, hd if mode else hd[0], mode, bounds=b, window=win)
            return ref, dref
        return pmap(one, range(len(self.specs)))


def test_c_every_staged_array_kind_on_three_budgets():
    budgets = {"1 MB": 1, "default": None, "512 MB": 512}
    launches = {}
    refs = None
    for name, mb in budgets.items():
        with host_budget_renderer(mb) as Rc:
            batch = Hetero(Rc, np.random.default_rng(2718))
            refs = refs or batch.references()
            raw, raw_d, _, launches[name] = batch.run(Rc, False, pinned=True)
            outs, outs_d, loud, _ = batch.run(Rc, True, pinned=False)
            key = "C %s" % name
            res = []
            for k, (label, mode, x, h, b, idx, w, win, direct) in enumerate(batch.specs):
                n0 = 0 if win is None else win[0]
                res.append(check(key, raw[k], refs[k][0], n0=n0, label="%s: %s" % (key, label)))
                if direct:
                    res.append(check(key, raw_d[k], refs[k][1], n0=n0, label="%s: %s direct" % (key, label)))
                t = batch.targets[k] if k < len(batch.targets) else None
                if t is None:
                    assert np.array_equal(outs[k], raw[k]), (key, label)
                    if direct:
                        assert np.array_equal(outs_d[k], raw_d[k]), (key, label)
                else:
                    check_loudness(key, raw[k], outs[k], loud[k][0], loud[k][1], t, "%s: %s" % (key, label),
                                   raw_d[k] if direct else None, outs_d[k] if direct else None)
            _noted(res)
            batch.bank.close()               # (its plans are gone: freed now, before its context)
    print("\nC: launches of the render without loudness per budget: %s" % launches)
    # 512 MB: one chunk holds every source, so every staged span sits next to every other kind in one slot (a chunk
    # launches at most k_blocks, k_rir_absmax, k_rir_direct, k_prepare and k_render); 1 MB: one slot per source or two
    assert launches["512 MB"] <= 5
    assert launches["1 MB"] > 2 * K_SLOTS * 2
    _report("C")


# ------------------------------------------------------------------------------------------------ D. growth
def _align(v, a):
    return (v + a - 1) // a * a


def ensure_cap(cap, need):
    """ensure()'s rule (csrc/ss_internal.h): grow to need + need / 4 in whole MB when need exceeds the capacity."""
    return cap if need <= cap else _align(need + need // 4, MB)


def out_need(C, N, n_e=None):
    """stage_source's d_out bytes of one whole source without a direct stem (n_e: its gating intervals when it has a
    loudness target)."""
    b = _align(4 * C * N, 256)
    if n_e is not None:
        b += _align(_align(8 * LOUD_SCRATCH_DOUBLES * C * n_e, 256), 256) + 256
    return b


def _n_e(N):
    from sonicsim_b200.SonicSim_audio import gating_plan
    return len(gating_plan(N, float(RATE), block_size_of(N, RATE))[0]) - 1


def test_d_growth_between_and_within_calls(bench_items, bench_refs):
    """A fresh context with a 1 MB host budget, so that every source of a call is a chunk of its own and chunk k takes
    slot k % 4: small, bench-sized, small again, then more items with new clip lengths in ascending size, so that
    chunks at k >= 4 regrow slots the same call's earlier chunks used.  Every call runs without and with loudness
    targets; a model of the slots' d_out capacities (stage_source's spans, ensure's rule) shows the reallocations."""
    render, _ = _R()
    rng = np.random.default_rng(99)
    small = [render.StaticSource(so.synth_dry(rng, 20000 + 3 * k), so.synth_rirs(rng, 1, 2, 4096 + 512)[0])
             for k in range(3)]
    small_refs = pmap(lambda s: reference(s.dry, s.rir, 0), small)
    bench_srcs = [render.MovingSource(x, h, b) for x, h, b in bench_items[:6]]
    lengths = [24011 + 70001 * k for k in range(10)]     # 24 011 .. 654 020 samples, ascending
    larger = []
    for k, N in enumerate(lengths):
        P = 6 + k
        h = so.synth_rirs(rng, P, 8, 4096)
        np.random.seed(k)
        larger.append(render.MovingSource(so.synth_dry(rng, N), h,
                                          render.trajectory_bounds(so.synth_path(rng, P), N)))
    larger_refs = pmap(lambda s: reference(s.dry, s.rirs, 1, bounds=s.bounds), larger)
    calls = [("small", small, small_refs), ("bench", bench_srcs, bench_refs[:6]), ("small again", small, small_refs),
             ("larger", larger, larger_refs)]
    caps = [0] * K_SLOTS
    grew = []
    with host_budget_renderer(1) as Rc:
        for ci, (name, srcs, refs) in enumerate(calls):
            targets = [-18.0 - 1.3 * k - ci for k in range(len(srcs))]
            for lufs in (False, True):
                outs = [Out(s.rirs.shape[1] if hasattr(s, "rirs") else s.rir.shape[0], len(s.dry), pinned=k % 3 != 1)
                        for k, s in enumerate(srcs)]
                plan = Rc.plan_host(srcs, [o.view() for o in outs], targets if lufs else None, RATE)
                plan.run()
                got = [o.get("D %s %d" % (name, k)) for k, o in enumerate(outs)]
                for k, (s, o) in enumerate(zip(srcs, outs)):
                    C, N = o.C, o.n
                    need = out_need(C, N, _n_e(N) if lufs else None)
                    new = ensure_cap(caps[k % K_SLOTS], need)
                    if new != caps[k % K_SLOTS]:
                        grew.append((name, lufs, k))
                    caps[k % K_SLOTS] = new
                if not lufs:
                    raw = got
                    _noted(pmap(lambda k: check("D growth", raw[k], refs[k], label="D %s stem %d" % (name, k)),
                                range(len(srcs))))
                else:
                    loud = plan.loudness()
                    for k in range(len(srcs)):
                        check_loudness("D growth", raw[k], got[k], loud[k][0], loud[k][1], targets[k],
                                       "D %s stem %d" % (name, k))
    print("\nD: chunks whose slot d_out regrew (call, loudness, chunk): %s" % grew)
    assert any(g[0] == "bench" for g in grew)
    assert any(g[0] == "larger" and g[2] >= K_SLOTS for g in grew)       # within one call, a slot used before
    _report("D growth")


def _lufs_host(Rc, x, target):
    """ss_lufs_norm_host over the (C, N) stem x in guarded pageable buffers: (LUFS, gain, output (C, N))."""
    from sonicsim_b200.SonicSim_audio import gating_plan
    C, N = x.shape
    block = block_size_of(N, RATE)
    brk, lo, hi = gating_plan(N, float(RATE), block)
    xin, out = Guard(x), Guard(n=C * N)
    lufs, gain = ctypes.c_double(np.nan), ctypes.c_double(np.nan)
    st = Rc.lib.ss_lufs_norm_host(Rc.ctx, xin.ptr, out.ptr, N, C, 1, N, float(RATE), block, target, brk.ctypes.data,
                                  len(brk) - 1, lo.ctypes.data, hi.ctypes.data, len(lo), ctypes.byref(lufs),
                                  ctypes.byref(gain))
    assert st == 0
    assert np.array_equal(xin.get(), x.reshape(-1))
    return lufs.value, gain.value, out.get().reshape(C, N)


def test_d_host_entries_through_growing_and_shrinking_scratch():
    """ss_lufs_norm_host, ss_mix_host_ex and ss_overlap_host share the first slot's input buffer: on a fresh context,
    sizes rising through several of ensure's MB steps and falling again, the three entries in turn."""
    sizes = [3001, 120007, 700001, 1900003, 4100005, 900001, 40001, 2501]       # samples per channel
    rng = np.random.default_rng(5)
    cap, steps = 0, []
    with host_budget_renderer(None) as Rc:
        scratch_doubles = int(Rc.lib.ss_mix_scratch_doubles())
        for E in sizes:
            # loudness: (2, E) stems, levels that differ by size
            x = (so.synth_dry(rng, 2 * E).reshape(2, E) * np.float32(0.3 + 0.1 * len(steps))).astype(np.float32)
            target = -17.0 - len(steps)
            lufs, gain, out = _lufs_host(Rc, x, target)
            check_loudness("D host entries", x, out, lufs, gain, target, "D lufs_norm_host E=%d" % E)
            # mixture: two speakers, one noise, an SIR and SNR of their own, a delayed noise on every other size
            spk = np.stack([so.synth_dry(rng, E), so.synth_dry(rng, E) * F32(0.25)]).astype(F32)
            noise = (so.synth_dry(rng, E) * F32(0.5))[None].astype(F32)
            sirs, snr, delay = np.array([1.5 - len(steps) % 3], F32), F32(5.0 + len(steps)), (len(steps) % 2) * 37
            gs, gn, gsir = Guard(spk), Guard(noise), Guard(sirs)
            mix, so_ = Guard(n=E), Guard(n=2 * E)
            st = Rc.lib.ss_mix_host_ex(Rc.ctx, gs.ptr, gn.ptr, gsir.ptr, float(snr), mix.ptr, so_.ptr, 2, 1, E, delay)
            assert st == 0
            assert np.array_equal(gs.get(), spk.reshape(-1)) and np.array_equal(gn.get(), noise.reshape(-1))
            c = SimpleNamespace(spk=spk, noise=noise, sirs=sirs, snr=snr, delay=delay, S=2, E=E)
            check_mix(c, mix.get(), so_.get().reshape(2, E))
            # overlap: three rows
            xo = so.synth_dry(rng, 3 * E).reshape(3, E)
            D = 1 + E // 7
            go, gy = Guard(xo), Guard(n=3 * E)
            assert Rc.lib.ss_overlap_host(Rc.ctx, go.ptr, gy.ptr, 3, E, D) == 0
            assert np.array_equal(gy.get().reshape(3, E), overlap_exact(xo, D)), E
            # the first slot's block of the mixture (speakers, noise, mix, SIRs, scratch) and of the overlap (x, y),
            # as ss_mix_host_ex and ss_overlap_host lay them out; the loudness block (the stem, its tables and scratch)
            # is the smallest of the three
            mix_need = _align(8 * E, 256) + 2 * _align(4 * E, 256) + 256 + _align(8 * scratch_doubles, 256)
            grown = None
            for need in (mix_need, 2 * _align(12 * E, 256)):
                new = ensure_cap(cap, need)
                grown = new // MB if new != cap else grown
                cap = new
            steps.append(grown)
    print("\nD: first-slot capacity after each size (MB, None: kept): %s" % steps)
    assert sum(s is not None for s in steps) >= 3 and steps[-1] is None
    _report("D host entries")


# ------------------------------------------------------------------------------------------------ E. drop-in
def test_e_dropin_at_full_configs1_size():
    from sonicsim_b200 import SonicSim_moving as sm
    rng = np.random.default_rng(2024)
    P, C, L, N = bench.CFG["P"], bench.CFG["C"], bench.CFG["L"], bench.CFG["N"]
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
    np.random.seed(2024)
    idx, w = sm.setup_dynamic_interp(pos, N)
    y = sm.convolve_moving_receiver(x, h, idx, w)
    h0 = so.synth_rirs(rng, 1, C, L)[0]
    yf = sm.convolve_fixed_receiver(x, h0)
    refs = pmap(lambda j: reference(x, h, 2, idx=idx, w=w) if j == 0 else reference(x, h0, 0), (0, 1))
    _noted([check("E drop-in moving", y, refs[0], label="convolve_moving_receiver"),
            check("E drop-in fixed", yf, refs[1], label="convolve_fixed_receiver")])
    _report("E")
