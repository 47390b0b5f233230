"""Every device entry point on a side stream whose earlier work is still queued, against float64.

Training code calls the library on a stream of its own (a prefetch stream, `with torch.cuda.stream(s)`), not on the
legacy default stream, so a dropped `stream` argument, a fork onto the context's internal streams that does not join
back, or a device value read ahead of the caller's write only shows up there.  Every case below follows one pattern on
s = torch.cuda.Stream() (never the legacy NULL stream):

1. on s, the outputs are filled with NaN and the inputs with poison;
2. torch.cuda._sleep queues about a quarter of a second of work on s;
3. the real inputs are written on s with copy_;
4. the call is made on s, and s must still be busy afterwards, so the call was enqueued behind the sleep;
5. still on s, with no synchronisation, every output is cloned;
6. after a synchronisation the clones are checked: stems sample by sample against tests/render_reference.py,
   mixtures against tests/mix_reference.py (gains within 3 ulps, the composition exact), loudness against the float64
   BS.1770 oracle to 1e-6 dB, dry streams against the polyphase reference of test_gpu_dry_kernel.py.

The first launch of a kernel in a process can block the host until the device is idle (lazy module loading), which
would wait out the sleep, so every case makes its calls once without the sleep first.  Poison is harmless if read early: dry samples, RIRs, stems and gains become NaN; window starts, pool picks and device
bounds tables become a different legal value, so a read before the write renders a valid but wrong crop, never a wild
index.  Cases: ss_render_dev in one chunk (serial on s) and in many (forked and joined); device plans as a graph, in a
context without graphs and with profiling on; banks and pools built behind the sleep and used at once by a plan on a
second stream; ss_mix_dev, ss_overlap_dev, ss_loudness_dev and ss_dry_assemble_dev; a render on s handed to a mixture
on another stream through the caller's event; host calls right after asynchronous device work on the same context
(their descriptor slots and scratch must wait for the device work still reading them); and a renderer on cuda:1 while
cuda:0 is current."""
import contextlib
import ctypes
import os

import numpy as np
import pytest
import torch

from direct_path import direct_path_rirs, normalized
from mix_reference import F32, compose_mix, f32_neighbours, mix_gains_f64, overlap_exact
from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from gpu_plumbing import small_host_budget_context
from loudness_cases import (EXACT_DB, Stem, _reference, _scene, _stem_shape, assert_clear_of_gates, block_size_of,
                            stems as loud_stems)
from mix_reference import Clip, DryBuf

pytestmark = pytest.mark.gpu

NAN = float("nan")
SLEEP = int(5e8)            # GPU cycles: about 0.25 s, far longer than the host work between the sleep and the query
SMALL = 1 << 20             # the smallest device chunk budget: about one source of render_batch per chunk
DEFAULT_CHUNK_BYTES = 32 << 20


def _lib_render():
    from sonicsim_b200 import _lib, render
    return _lib, render, render.default_renderer()


def to_device(a, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def side_stream(device=None):
    s = torch.cuda.Stream(device=device)
    assert s.cuda_stream != 0                         # not the legacy default stream
    return s


def stage(s, outs, writes):
    """Steps 1-3 on stream s: every tensor of `outs` NaN, every (dst, real, poison) of `writes` poisoned, a sleep, the
    real values.  `real` and a tensor `poison` are complete before s starts (made on the default stream)."""
    torch.cuda.synchronize()
    with torch.cuda.stream(s):
        for o in outs:
            o.fill_(NAN)
        for dst, _, p in writes:
            if isinstance(p, torch.Tensor):
                dst.copy_(p)
            else:
                dst.fill_(p)
        torch.cuda._sleep(SLEEP)
        for dst, real, _ in writes:
            dst.copy_(real)


def unstaged(writes):
    """The real values of `writes` on the default stream, complete on return: the inputs of a warm-up call."""
    for dst, real, _ in writes:
        dst.copy_(real)
    torch.cuda.synchronize()


def snapshot(s, outs, busy=()):
    """Steps 4-6: s (and every stream of `busy`) still has the sleep queued; clones of `outs` on s, then synchronise.
    Returns the clones as NumPy arrays."""
    for q in (s,) + tuple(busy):
        assert not q.query(), "the call was not enqueued behind the queued work: the case proves nothing"
    with torch.cuda.stream(s):
        snaps = [o.clone() for o in outs]
    torch.cuda.synchronize()
    return [c.cpu().numpy() for c in snaps]


def grow_ring(lib, ctx):
    """Grow every descriptor-ring slot of `ctx` past what the cases here describe, so that no call below reallocates
    a slot (a reallocation synchronises the device and would wait out the sleep): one ss_dry_assemble_dev of 4096
    empty clips per slot, on the default stream."""
    from sonicsim_b200 import _lib
    src, out = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    clip = _lib.SsDryClip(src=src.data_ptr(), kernel_t=None, dst_start=0, src_start=0, count=0, channels=1, src_len=1,
                          orig=1, new_rate=1, width=0, taps=1)
    arr = (_lib.SsDryClip * 4096)(*([clip] * 4096))
    for _ in range(8):                                # kRing = 6 slots
        _lib.check(lib.ss_dry_assemble_dev(ctx, arr, 4096, ctypes.c_void_p(out.data_ptr()), 1, None))
    torch.cuda.synchronize()


def legal_bounds(rng, N, P):
    """A random ascending bounds table from 0 to N with P entries and no empty segment."""
    inner = np.sort(rng.choice(np.arange(1, N), P - 2, replace=False))
    return np.concatenate([[0], inner, [N]]).astype(np.int32)


def other_start(rng, a, hi):
    """A legal start in [0, hi] other than a (the poison of a start tensor)."""
    b = int(rng.integers(0, hi + 1))
    return b if b != a else (a + 1 if a < hi else a - 1)


class Source:
    """One source with device bounds (moving) or none (static): NumPy inputs for float64, device tensors that stage()
    rewrites, its outputs, and its window: None (whole stem), ("fixed", start, n) or ("moving", n) with a device start."""

    def __init__(self, R, rng, static=False, N=20000, P=5, C=2, L=600, normalize=False, taps=0, window=None,
                 device="cuda"):
        self.rng, self.static, self.N, self.C, self.normalize, self.taps = rng, static, N, C, normalize, taps
        self.P = 1 if static else P
        self.x = so.synth_dry(rng, N)
        self.h = so.synth_rirs(rng, self.P, C, L)
        self.bounds = None if static else legal_bounds(rng, N, P)
        self.h_ref = normalized(self.h) if normalize else self.h
        self.h_dir = direct_path_rirs(self.h_ref, taps) if taps else None
        self.window = window
        self.n = N if window is None else window[-1]
        self.a = 0 if window is None or window[0] == "moving" else window[1]
        self.dev = device
        self.dx = torch.empty(N, device=device)
        self.dh = torch.empty(self.h.shape, device=device)
        self.db = None if static else torch.empty(P, dtype=torch.int32, device=device)
        self.start = torch.zeros(1, dtype=torch.int32, device=device) if window and window[0] == "moving" else None
        self.out = torch.empty((C, self.n), device=device)
        self.dout = torch.empty((C, self.n), device=device) if taps else None

    def writes(self):
        """(dst, real, poison) of every input; draws a new start for a moving window."""
        w = [(self.dx, to_device(self.x, self.dev), NAN), (self.dh, to_device(self.h, self.dev), NAN)]
        if not self.static:
            linear = np.round(np.linspace(0, self.N, self.P)).astype(np.int32)
            w.append((self.db, to_device(self.bounds, self.dev), to_device(linear, self.dev)))
        if self.start is not None:
            hi = self.N - self.n
            self.a = int(self.rng.integers(0, hi + 1))
            w.append((self.start, to_device(np.array([self.a], np.int32), self.dev),
                      to_device(np.array([other_start(self.rng, self.a, hi)], np.int32), self.dev)))
        return w

    def outs(self):
        return [self.out] + ([self.dout] if self.taps else [])

    def py(self):
        from sonicsim_b200 import render
        win = None
        if self.window is not None:
            win = (self.start[0], self.n) if self.window[0] == "moving" else (self.a, self.n)
        if self.static:
            return render.StaticSource(self.dx, self.dh[0], self.normalize, self.taps, win)
        return render.MovingSource(self.dx, self.dh, self.db, None, self.normalize, self.taps, win)

    def check(self, y, direct=False, label=""):
        h = self.h_dir if direct else self.h_ref
        y64, scale = render_check_inputs(self.x, h, 0 if self.static else 1, bounds=self.bounds,
                                         window=None if self.window is None else (self.a, self.n))
        check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=self.a, label=label)


def render_batch(R, rng):
    """Moving sources (whole, fixed and moving windows; RIR normalisation and direct stems on some) and a static one:
    at most 6 chunks, so that a forked render does not wrap the 6-slot descriptor ring, whose pinned blocks are reused
    only after their earlier copies (a wrap would block the host until the sleep is over)."""
    srcs = []
    for j in range(5):
        win = (None, ("fixed", 3001, 5000), ("moving", 6000))[j % 3]
        srcs.append(Source(R, rng, C=4, normalize=j % 2 == 0, taps=40 if j % 3 != 1 else 0, window=win))
    srcs.append(Source(R, rng, static=True, C=4, normalize=True, taps=40, window=("moving", 7000)))
    return srcs


def render_dev_on(R, s, srcs):
    """Stage every source on s and render the batch there with render_device (torch's current stream: s)."""
    writes = [w for x in srcs for w in x.writes()]
    stage(s, [o for x in srcs for o in x.outs()], writes)
    with torch.cuda.stream(s):
        R.render_device([x.py() for x in srcs], [x.out for x in srcs], direct_outs=[x.dout for x in srcs])


def check_stems(srcs, snaps, what):
    k = 0
    for i, x in enumerate(srcs):
        x.check(snaps[k], label="%s source %d" % (what, i))
        k += 1
        if x.taps:
            x.check(snaps[k], direct=True, label="%s source %d direct" % (what, i))
            k += 1
    return snaps[k:]


def warm(R, srcs):
    """One render of the batch on the default stream: the context's scratch is grown before any staged call."""
    for w in (w for x in srcs for w in x.writes()):
        w[0].copy_(w[1])
    R.render_device([x.py() for x in srcs], [x.out for x in srcs], direct_outs=[x.dout for x in srcs])
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ ss_render_dev
@pytest.mark.parametrize("chunks", ["one", "many"])
def test_render_dev_on_a_side_stream(chunks):
    """One chunk runs serially on s; many chunks fork onto the context's streams and must join back into s before the
    clones.  Whole stems, fixed windows and moving windows whose starts are written behind the sleep."""
    _lib, render, R = _lib_render()
    R.set_chunk_bytes(SMALL if chunks == "many" else 1 << 30)
    try:
        grow_ring(R.lib, R.ctx)
        srcs = render_batch(R, np.random.default_rng(11))
        warm(R, srcs)
        s = side_stream()
        for run in range(2):
            R.reset_stats()
            render_dev_on(R, s, srcs)
            launches = R.launch_count()
            snaps = snapshot(s, [o for x in srcs for o in x.outs()])
            # one chunk: at most k_blocks, k_rir_absmax, k_rir_direct, k_prepare and k_render; many: at least four
            # chunks of at least k_blocks, k_prepare and k_render each (every source here has device tables)
            assert (launches <= 5) if chunks == "one" else (launches >= 4 * 3), launches
            check_stems(srcs, snaps, "%s chunk(s), run %d" % (chunks, run))
    finally:
        R.set_chunk_bytes(DEFAULT_CHUNK_BYTES)


# ------------------------------------------------------------------------------------------------ device plans
@contextlib.contextmanager
def renderer_for(mode):
    """The default renderer (graph; profiling switched on and off), or one whose own context runs plans without graphs
    (SS_NO_GRAPH is read by ss_create), with a device chunk budget of SMALL."""
    _lib, render, R = _lib_render()
    if mode != "no_graph":
        R.set_chunk_bytes(SMALL)
        R.set_profiling(mode == "profiling")
        try:
            yield R
        finally:
            R.set_profiling(False)
            R.set_chunk_bytes(DEFAULT_CHUNK_BYTES)
        return
    old = os.environ.get("SS_NO_GRAPH")
    os.environ["SS_NO_GRAPH"] = "1"
    ctx = ctypes.c_void_p()
    try:
        assert R.lib.ss_create(R.device, ctypes.byref(ctx)) == 0
    finally:
        if old is None:
            del os.environ["SS_NO_GRAPH"]
        else:
            os.environ["SS_NO_GRAPH"] = old
    R2 = render.Renderer.__new__(render.Renderer)
    R2.lib, R2.device, R2.ctx = R.lib, R.device, ctx
    R2.set_chunk_bytes(SMALL)
    try:
        yield R2
    finally:
        torch.cuda.synchronize()
        R.lib.ss_destroy(ctx)


class Candidate:
    """A banked static candidate of a pool; its dry signal is staged like a source's."""

    def __init__(self, R, rng, N, C=2, L=600):
        from sonicsim_b200 import render
        self.x, self.h = so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, L)
        self.dx = to_device(self.x)
        self.th = to_device(self.h[0])
        self.bank = R.rir_bank(self.th)
        self.src = render.StaticSource(self.dx, self.bank)

    def check(self, y, a, n, label):
        y64, scale = render_check_inputs(self.x, self.h, 0, window=(a, n))
        check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=a, label=label)


def check_mixture(spk, noise, sirs, snr, mix, spk_out, label):
    """spk (S, E), noise (M, E): every gain within 3 ulps of mix_gains_f64, mix and spk_out exactly compose_mix."""
    g64, gn64 = mix_gains_f64(spk, noise, sirs, snr)
    assert np.array_equal(spk_out[0], spk[0]), label
    g = [F32(1.0)]
    for k in range(1, spk.shape[0]):
        fits = [v for v in f32_neighbours(g64[k]) if np.array_equal(spk_out[k], spk[k] * v)]
        assert fits, (label, "speaker %d: no float32 gain within 3 ulps" % k, g64[k])
        g.append(fits[0])
    g = np.array(g, F32)
    fits = [v for v in f32_neighbours(gn64) if np.array_equal(mix, compose_mix(spk, noise, g, v)[0])]
    assert fits, (label, "no noise gain within 3 ulps", gn64)
    assert np.array_equal(spk_out, compose_mix(spk, noise, g, fits[0])[1]), label


@pytest.mark.parametrize("mode", ["graph", "no_graph", "profiling"])
def test_plan_runs_on_a_side_stream(mode):
    """A plan of several chunks: four moving windows (raw RIRs, normalised and direct on two) and two pooled slots
    whose starts, picks, SIRs, SNRs, dry signals and RIRs are all written behind the sleep, with two mixtures.  Two
    runs, each with new values."""
    from sonicsim_b200 import render
    rng = np.random.default_rng({"graph": 1, "no_graph": 2, "profiling": 3}[mode])
    T = 8000
    with renderer_for(mode) as R:
        cands = [Candidate(R, rng, 12000 + 1999 * j) for j in range(3)]
        pool = R.source_pool([c.src for c in cands])
        srcs = [Source(R, rng, normalize=j < 2, taps=40 if j < 2 else 0, window=("moving", T)) for j in range(4)]
        picks = torch.zeros(2, dtype=torch.int32, device="cuda")
        pstart = torch.zeros(2, dtype=torch.int32, device="cuda")
        pouts = [torch.empty((2, T), device="cuda") for _ in range(2)]
        sirs = torch.zeros((2, 1), device="cuda")
        snr = torch.zeros(2, device="cuda")
        mix = torch.empty((2, 2, T), device="cuda")
        spk_out = torch.empty((2, 2, 2, T), device="cuda")
        items = [x.py() for x in srcs] + [render.Pooled(pool, picks[j], (pstart[j], T)) for j in range(2)]
        outs = [x.out for x in srcs] + pouts
        mixtures = [render.Mixture([2 * u, 2 * u + 1], [4 + u], sirs[u], snr[u], mix[u], spk_out[u]) for u in range(2)]
        plan = R.plan_device(items, outs, direct_outs=[x.dout for x in srcs] + [None, None], mixtures=mixtures)
        s = side_stream()
        n_min = min(c.x.size for c in cands)
        try:
            unstaged([w for x in srcs for w in x.writes()])
            plan.run()                                    # warm-up (and, in graph mode, the capture)
            torch.cuda.synchronize()
            for run in range(2):
                pk = [int(v) for v in rng.integers(0, 3, 2)]
                ps = [int(v) for v in rng.integers(0, n_min - T + 1, 2)]
                sv, nv = rng.uniform(-6, 6, (2, 1)).astype(np.float32), rng.uniform(10, 20, 2).astype(np.float32)
                writes = [w for x in srcs for w in x.writes()]
                writes += [(c.dx, to_device(c.x), NAN) for c in cands]
                writes += [(picks, to_device(np.array(pk, np.int32)), to_device(np.array([(v + 1) % 3 for v in pk], np.int32))),
                           (pstart, to_device(np.array(ps, np.int32)),
                            to_device(np.array([other_start(rng, a, n_min - T) for a in ps], np.int32))),
                           (sirs, to_device(sv), NAN), (snr, to_device(nv), NAN)]
                snap_outs = [o for x in srcs for o in x.outs()] + pouts + [mix, spk_out]
                stage(s, snap_outs, writes)
                R.reset_stats()
                with torch.cuda.stream(s):
                    plan.run()
                launches = R.launch_count()
                snaps = snapshot(s, snap_outs)
                assert launches >= 2 * 3 + 4, launches                # several chunks, then the mixtures
                assert plan.is_graph() == (mode == "graph")
                what = "%s run %d" % (mode, run)
                rest = check_stems(srcs, snaps, what)
                for j in range(2):
                    cands[pk[j]].check(rest[j], ps[j], T, "%s pooled slot %d (candidate %d)" % (what, j, pk[j]))
                m, so_ = rest[2], rest[3]
                stem = {0: snaps[0], 1: snaps[2], 2: snaps[4], 3: snaps[5], 4: rest[0], 5: rest[1]}
                for u in range(2):
                    spk = np.stack([stem[2 * u].reshape(-1), stem[2 * u + 1].reshape(-1)])
                    check_mixture(spk, stem[4 + u].reshape(1, -1), sv[u], nv[u], m[u].reshape(-1),
                                  so_[u].reshape(2, -1), "%s mixture %d" % (what, u))
            R.check_device_errors()
        finally:
            plan.close()
            pool.close()
            for c in cands:
                c.bank.close()


def test_banks_and_pool_built_behind_queued_work_serve_a_plan_on_another_stream():
    """RIR tensors written behind the sleep on s, banks built from them there (and the tensors NaN-filled right after,
    still on s), a pool over those banks, then at once a plan over the pool and one more banked source run on a second
    stream s2: the run waits for the banks and the pool's `ready` event, recorded from a non-default stream."""
    _lib, render, R = _lib_render()
    rng = np.random.default_rng(21)
    T, C, L = 6000, 2, 600
    xs = [so.synth_dry(rng, 15000 + 1000 * j) for j in range(4)]
    hs = [so.synth_rirs(rng, 1, C, L) for _ in range(3)]
    hm = so.synth_rirs(rng, 4, C, L)
    N3 = xs[3].size
    bm = legal_bounds(rng, N3, 4)
    dxs = [to_device(x) for x in xs]
    dbm = to_device(bm)
    ths = [torch.empty((C, L), device="cuda") for _ in range(3)]
    thm = torch.empty((4, C, L), device="cuda")
    writes = [(t, to_device(h[0]), NAN) for t, h in zip(ths, hs)] + [(thm, to_device(hm), NAN)]
    for staged in (False, True):                          # a warm-up on the default stream, then the case
        s, s2 = (side_stream(), side_stream()) if staged else (torch.cuda.default_stream(),) * 2
        if staged:
            stage(s, [], writes)
        else:
            unstaged(writes)
        with torch.cuda.stream(s):
            banks = [R.rir_bank(t) for t in ths] + [R.rir_bank(thm)]
            for t in ths + [thm]:
                t.fill_(NAN)                              # after the banks' kernels: a bank never reads its RIRs again
        pool = R.source_pool([render.StaticSource(dxs[j], banks[j]) for j in range(3)])
        pick = torch.zeros(1, dtype=torch.int32, device="cuda")
        pout, mout = torch.empty((C, T), device="cuda"), torch.empty((C, N3), device="cuda")
        plan = R.plan_device([render.Pooled(pool, pick[0], (1234, T)),
                              render.MovingSource(dxs[3], banks[3], dbm, bm)], [pout, mout])
        try:
            with torch.cuda.stream(s2):
                pick.fill_(2)
                pout.fill_(NAN)
                mout.fill_(NAN)
                plan.run()
            if staged:
                y_pool, y_mov = snapshot(s2, [pout, mout], busy=(s,))
            else:
                torch.cuda.synchronize()
                y_pool, y_mov = pout.cpu().numpy(), mout.cpu().numpy()
            what = "staged" if staged else "warm-up"
            y64, scale = render_check_inputs(xs[3], hm, 1, bounds=bm)
            check_render(y_mov, y64, scale, TAU_LOCAL, TAU_GLOBAL, label="%s banked moving source" % what)
            y64, scale = render_check_inputs(xs[2], hs[2], 0, window=(1234, T))
            check_render(y_pool, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=1234, label="%s pooled slot" % what)
        finally:
            plan.close()
            pool.close()
            for b in banks:
                b.close()


# ------------------------------------------------------------------------------------------------ C ABI, one call each
def _stream(s):
    return ctypes.c_void_p(s.cuda_stream)


def test_mix_dev_on_a_side_stream():
    from sonicsim_b200 import _lib
    _, _, R = _lib_render()
    grow_ring(R.lib, R.ctx)
    rng = np.random.default_rng(31)
    cases = [(3, 2, 48001, 12.0), (2, 1, 65536, -3.0)]              # scalar path (odd E) and float4 path
    bufs, writes, outs, items = [], [], [], []
    scr_n = int(R.lib.ss_mix_scratch_doubles())
    for S, M, E, snr in cases:
        spk = (rng.standard_normal((S, E)) * 0.1).astype(F32)
        noi = (rng.standard_normal((M, E)) * 0.05).astype(F32)
        sirs = rng.uniform(-6, 6, S - 1).astype(F32)
        t_spk, t_noi, t_sir = torch.empty((S, E), device="cuda"), torch.empty((M, E), device="cuda"), \
            torch.empty(S - 1, device="cuda")
        t_mix, t_out = torch.empty(E, device="cuda"), torch.empty((S, E), device="cuda")
        scr = torch.empty(scr_n, dtype=torch.float64, device="cuda")
        writes += [(t_spk, to_device(spk), NAN), (t_noi, to_device(noi), NAN), (t_sir, to_device(sirs), NAN)]
        outs += [t_mix, t_out]
        bufs.append((spk, noi, sirs, snr, t_spk, t_noi, t_sir, scr))
        items.append(_lib.SsMixItem(speakers=t_spk.data_ptr(), noises=t_noi.data_ptr(), sirs=t_sir.data_ptr(),
                                    mix=t_mix.data_ptr(), speakers_out=t_out.data_ptr(), scratch=scr.data_ptr(),
                                    E=E, S=S, M=M, snr=snr, noise_delay=0))
    arr = (_lib.SsMixItem * len(items))(*items)
    unstaged(writes)
    _lib.check(R.lib.ss_mix_dev(R.ctx, arr, len(items), None))          # warm-up
    s = side_stream()
    stage(s, outs, writes)
    _lib.check(R.lib.ss_mix_dev(R.ctx, arr, len(items), _stream(s)))
    snaps = snapshot(s, outs)
    for k, (spk, noi, sirs, snr, *_) in enumerate(bufs):
        check_mixture(spk, noi, sirs, snr, snaps[2 * k], snaps[2 * k + 1], "ss_mix_dev item %d" % k)


def test_overlap_dev_on_a_side_stream():
    _, _, R = _lib_render()
    rng = np.random.default_rng(32)
    rows, T, D = 3, 40001, 1777
    x = rng.standard_normal((rows, T)).astype(F32)
    tx, ty = torch.empty((rows, T), device="cuda"), torch.empty((rows, T), device="cuda")
    unstaged([(tx, to_device(x), NAN)])
    assert R.lib.ss_overlap_dev(R.ctx, ctypes.c_void_p(tx.data_ptr()), ctypes.c_void_p(ty.data_ptr()), rows, T, D,
                                None) == 0                                  # warm-up
    s = side_stream()
    stage(s, [ty], [(tx, to_device(x), NAN)])
    assert R.lib.ss_overlap_dev(R.ctx, ctypes.c_void_p(tx.data_ptr()), ctypes.c_void_p(ty.data_ptr()), rows, T, D,
                                _stream(s)) == 0
    [y] = snapshot(s, [ty])
    assert np.array_equal(y, overlap_exact(x, D))


def _loud_stems(sr=16000):
    """Two stems (C = 2 and 5) on the device, measured and normalised into separate buffers (one unaligned)."""
    out = []
    for k, (N, C) in enumerate(((52001, 2), (30000, 5))):
        x = loud_stems(40 + k, N, C, sr)
        assert_clear_of_gates(x, sr, block_size_of(N, sr))
        out.append(Stem(x, sr, -24.0 + 3 * k, "cn", "sep", off=k))
    torch.cuda.synchronize()
    return out


def _loud_stage(stems_):
    """(outputs, writes) of the loudness stems: outputs and results NaN, the input data poisoned with NaN."""
    outs, writes = [], []
    for st in stems_:
        outs += [st.obuf, st.res]
        writes.append((st.buf[st.off:st.off + st.n], st.buf[st.off:st.off + st.n].clone(), NAN))
    return outs, writes


def _loud_check(stems_, snaps, what):
    for k, st in enumerate(stems_):
        ob, res = snaps[2 * k], snaps[2 * k + 1]
        lufs, gain = float(res[0]), float(res[1])
        ref = _reference(st.x, st.sr)
        assert abs(lufs - ref) <= EXACT_DB, (what, k, lufs, ref)
        assert gain == pytest.approx(10 ** ((st.target - lufs) / 20), rel=1e-13), (what, k)
        y = ob[st.off:st.off + st.n].reshape(st.C, st.N).T
        assert np.array_equal(y, np.float32(gain) * st.x), (what, k)


def test_loudness_dev_on_a_side_stream():
    from sonicsim_b200 import _lib
    _, _, R = _lib_render()
    grow_ring(R.lib, R.ctx)
    st = _loud_stems()
    outs, writes = _loud_stage(st)
    arr = (_lib.SsLoudItem * len(st))(*[x.item for x in st])
    _lib.check(R.lib.ss_loudness_dev(R.ctx, arr, len(st), None))         # warm-up
    s = side_stream()
    stage(s, outs, writes)
    _lib.check(R.lib.ss_loudness_dev(R.ctx, arr, len(st), _stream(s)))
    _loud_check(st, snapshot(s, outs), "ss_loudness_dev")


def test_dry_assemble_dev_on_a_side_stream():
    from sonicsim_b200 import _lib
    _, _, R = _lib_render()
    grow_ring(R.lib, R.ctx)
    rng = np.random.default_rng(33)
    clips, cursor = [], 0
    for k, (orig, ch, L) in enumerate(((44100, 2, 30011), (16000, 1, 9000), (8000, 2, 4801), (48000, 1, 20000))):
        c = Clip((rng.standard_normal((ch, L)) * 0.1).astype(F32), orig, 16000, 0, 0, cursor, off=k % 4)
        n = c.count = -(-16000 * L // orig)
        c.c.count = n
        clips.append(c)
        cursor += n + 5
    out = DryBuf(cursor)
    torch.cuda.synchronize()
    writes = [(c.src.t[c.src.lo:c.src.lo + c.src.n], c.src.t[c.src.lo:c.src.lo + c.src.n].clone(), NAN)
              for c in clips]
    arr = (_lib.SsDryClip * len(clips))(*[c.c for c in clips])
    _lib.check(R.lib.ss_dry_assemble_dev(R.ctx, arr, len(clips), ctypes.c_void_p(out.ptr), out.n, None))   # warm-up
    s = side_stream()
    stage(s, [out.t[out.lo:out.lo + out.n]], writes)
    _lib.check(R.lib.ss_dry_assemble_dev(R.ctx, arr, len(clips), ctypes.c_void_p(out.ptr), out.n, _stream(s)))
    [y] = snapshot(s, [out.t[out.lo:out.lo + out.n]])
    placed = np.zeros(out.n, bool)
    for c in clips:
        got = y[c.dst_start:c.dst_start + c.count]
        placed[c.dst_start:c.dst_start + c.count] = True
        want, bound = c.expected()
        if bound is None:                                 # no resampling: exact
            assert np.array_equal(got, want), (c.orig, c.ch, c.L)
        else:
            assert np.all(np.abs(got.astype(np.float64) - want) <= bound), (c.orig, c.ch, c.L)
    assert not y[~placed].any()


# ------------------------------------------------------------------------------------------------ across streams
def test_render_on_one_stream_mixed_on_another_through_the_callers_event():
    """render_device on s (explicit stream argument) renders two speakers and a noise into one batch tensor; the caller
    records an event on s, a second stream s2 waits on it and ss_mix_dev mixes the stems there."""
    from sonicsim_b200 import _lib
    _, render, R = _lib_render()
    grow_ring(R.lib, R.ctx)
    rng = np.random.default_rng(41)
    T = 9000
    srcs = [Source(R, rng, window=("moving", T)), Source(R, rng, normalize=True, window=("fixed", 2222, T)),
            Source(R, rng, static=True, window=("moving", T))]
    spk, noi = torch.empty((2, 2, T), device="cuda"), torch.empty((1, 2, T), device="cuda")
    for x, o in zip(srcs, (spk[0], spk[1], noi[0])):
        x.out = o
    warm(R, srcs)
    sirs = torch.empty(1, device="cuda")
    mix, spk_out = torch.empty(2 * T, device="cuda"), torch.empty((2, 2 * T), device="cuda")
    scr = torch.empty(int(R.lib.ss_mix_scratch_doubles()), dtype=torch.float64, device="cuda")
    item = _lib.SsMixItem(speakers=spk.data_ptr(), noises=noi.data_ptr(), sirs=sirs.data_ptr(), mix=mix.data_ptr(),
                          speakers_out=spk_out.data_ptr(), scratch=scr.data_ptr(), E=2 * T, S=2, M=1, snr=14.5,
                          noise_delay=0)
    s, s2 = side_stream(), side_stream()
    sv = np.array([2.5], np.float32)
    unstaged([(sirs, to_device(sv), NAN)])
    _lib.check(R.lib.ss_mix_dev(R.ctx, ctypes.byref(item), 1, None))      # warm-up
    stage(s, [spk, noi, mix, spk_out], [w for x in srcs for w in x.writes()] + [(sirs, to_device(sv), NAN)])
    R.render_device([x.py() for x in srcs], [x.out for x in srcs], stream=s.cuda_stream)
    ev = torch.cuda.Event()
    ev.record(s)
    s2.wait_event(ev)
    _lib.check(R.lib.ss_mix_dev(R.ctx, ctypes.byref(item), 1, _stream(s2)))
    y_spk, y_noi, y_mix, y_out = snapshot(s2, [spk, noi, mix, spk_out], busy=(s,))
    for x, y in zip(srcs, (y_spk[0], y_spk[1], y_noi[0])):
        x.check(y, label="stem")
    check_mixture(y_spk.reshape(2, -1), y_noi.reshape(1, -1), sv, F32(14.5), y_mix, y_out, "mixture on s2")


# ------------------------------------------------------------------------------------------------ host calls
def _host(x):
    """The NumPy source of a Source for render_host (bounds on the host)."""
    from sonicsim_b200 import render
    if x.static:
        return render.StaticSource(x.x, x.h[0], x.normalize, x.taps)
    return render.MovingSource(x.x, x.h, x.bounds, None, x.normalize, x.taps)


def test_render_host_right_after_render_dev_on_a_side_stream():
    """A forked ss_render_dev on s, still queued behind the sleep, then at once render_host on the same context: its
    chunks take descriptor slots and scratch that the device render's chunks are still to read."""
    _, render, R = _lib_render()
    R.set_chunk_bytes(SMALL)
    try:
        grow_ring(R.lib, R.ctx)
        srcs = render_batch(R, np.random.default_rng(51))
        hsrcs = [Source(R, np.random.default_rng(52 + j), normalize=j == 0, taps=40 if j == 0 else 0) for j in range(3)]
        hsrcs.append(Source(R, np.random.default_rng(55), static=True))
        warm(R, srcs)
        d = [np.empty((x.C, x.N), np.float32) if x.taps else None for x in hsrcs]
        R.render_host([_host(x) for x in hsrcs], direct_outs=d)
        s = side_stream()
        R.reset_stats()
        render_dev_on(R, s, srcs)
        assert R.launch_count() >= 4 * 3
        outs = [o for x in srcs for o in x.outs()]
        assert not s.query()
        with torch.cuda.stream(s):
            snaps = [o.clone() for o in outs]
        d = [np.full((x.C, x.N), np.nan, np.float32) if x.taps else None for x in hsrcs]
        res = R.render_host([_host(x) for x in hsrcs], direct_outs=d)
        torch.cuda.synchronize()
        check_stems(srcs, [c.cpu().numpy() for c in snaps], "render_dev")
        for j, x in enumerate(hsrcs):
            x.check(res[j], label="render_host source %d" % j)
            if x.taps:
                x.check(d[j], direct=True, label="render_host source %d direct" % j)
    finally:
        R.set_chunk_bytes(DEFAULT_CHUNK_BYTES)


def test_render_host_ex_right_after_mix_and_loudness_on_a_side_stream():
    """ss_mix_dev and ss_loudness_dev on s behind the sleep, then at once ss_render_host_ex on the same context with a
    1 MB host budget: many chunks with loudness targets, direct stems on three of them and chunks without targets in
    between, so its loudness calls on the side streams and its renders on the compute stream take the ring's slots in
    an order that reuses every slot on another stream than the one that used it last.  The host-path loudness matches
    the oracle to 1e-6 dB and each direct stem takes its reverberant stem's gain; the device calls' results match
    theirs."""
    from sonicsim_b200 import _lib
    _, render, R = _lib_render()
    rng = np.random.default_rng(61)
    srcs, targets, _ = _scene(np.random.default_rng(85), 12)
    direct = (1, 4, 8)
    for i in direct:
        srcs[i] = srcs[i]._replace(direct_taps=40)
    assert all(targets[i] is not None for i in direct)
    st = _loud_stems()
    S, M, E = 3, 2, 30001
    spk = (rng.standard_normal((S, E)) * 0.1).astype(F32)
    noi = (rng.standard_normal((M, E)) * 0.05).astype(F32)
    sv = rng.uniform(-6, 6, S - 1).astype(F32)
    t_spk, t_noi, t_sir = torch.empty((S, E), device="cuda"), torch.empty((M, E), device="cuda"), \
        torch.empty(S - 1, device="cuda")
    t_mix, t_out = torch.empty(E, device="cuda"), torch.empty((S, E), device="cuda")
    scr = torch.empty(int(R.lib.ss_mix_scratch_doubles()), dtype=torch.float64, device="cuda")
    item = _lib.SsMixItem(speakers=t_spk.data_ptr(), noises=t_noi.data_ptr(), sirs=t_sir.data_ptr(),
                          mix=t_mix.data_ptr(), speakers_out=t_out.data_ptr(), scratch=scr.data_ptr(), E=E, S=S, M=M,
                          snr=11.0, noise_delay=0)
    larr = (_lib.SsLoudItem * len(st))(*[x.item for x in st])
    with small_host_budget_context() as ctx:
        grow_ring(R.lib, ctx)

        def host_ex(lufs_targets):
            outs = [np.full(_stem_shape(x), np.nan, np.float32) for x in srcs]
            dd = [np.full(_stem_shape(x), np.nan, np.float32) if i in direct else None for i, x in enumerate(srcs)]
            plan = R.plan_host(srcs, outs, lufs_targets, 16000, dd)
            if plan.post is None:
                _lib.check(R.lib.ss_render_host(ctx, plan.items, plan.n))
            else:
                _lib.check(R.lib.ss_render_host_ex(ctx, plan.items, plan.n, plan.post))
            return outs, dd, plan.loudness()
        R.lib.ss_reset_stats(ctx)
        raw, raw_d, _ = host_ex(None)
        # k_prepare and k_render per host-path chunk, plus k_rir_direct in the chunks of direct stems
        n_chunks = (R.lib.ss_launch_count(ctx) - len(direct)) // 2
        assert n_chunks >= 7, n_chunks
        warm_outs, _, _ = host_ex(targets)                        # grows the host path's buffers before the staged run
        loud_outs, loud_writes = _loud_stage(st)
        dev_outs = [t_mix, t_out] + loud_outs
        mix_writes = [(t_spk, to_device(spk), NAN), (t_noi, to_device(noi), NAN), (t_sir, to_device(sv), NAN)]
        unstaged(mix_writes)
        _lib.check(R.lib.ss_mix_dev(ctx, ctypes.byref(item), 1, None))                # warm-ups
        _lib.check(R.lib.ss_loudness_dev(ctx, larr, len(st), None))
        torch.cuda.synchronize()
        s = side_stream()
        stage(s, dev_outs, mix_writes + loud_writes)
        _lib.check(R.lib.ss_mix_dev(ctx, ctypes.byref(item), 1, _stream(s)))
        _lib.check(R.lib.ss_loudness_dev(ctx, larr, len(st), _stream(s)))
        assert not s.query()
        with torch.cuda.stream(s):
            snaps = [o.clone() for o in dev_outs]
        outs, dd, loud = host_ex(targets)
        torch.cuda.synchronize()
    snaps = [c.cpu().numpy() for c in snaps]
    check_mixture(spk, noi, sv, F32(11.0), snaps[0], snaps[1], "ss_mix_dev before render_host_ex")
    _loud_check(st, snaps[2:], "ss_loudness_dev before render_host_ex")
    for i, (x, t) in enumerate(zip(srcs, targets)):
        assert np.array_equal(outs[i], warm_outs[i]), i
        if t is None:
            assert np.array_equal(outs[i], raw[i]) and all(np.isnan(loud[i]))
            continue
        lufs, gain = loud[i]
        stem = np.ascontiguousarray(raw[i].T)
        ref = _reference(stem, 16000)
        assert abs(lufs - ref) <= EXACT_DB, (i, lufs, ref)
        assert gain == pytest.approx(10 ** ((t - lufs) / 20), rel=1e-13)
        assert np.array_equal(outs[i], np.float32(gain) * raw[i]), i
        if i in direct:
            assert np.array_equal(dd[i], np.float32(gain) * raw_d[i]), i     # the reverberant stem's gain


# ------------------------------------------------------------------------------------------------ another device
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_renderer_on_cuda1_while_cuda0_is_current():
    """A renderer on cuda:1 takes torch's current stream of cuda:1, not of the current device, for render_device and
    DevicePlan.run: both run behind queued work on a side stream of cuda:1 while cuda:0 is current."""
    from sonicsim_b200 import render
    R1 = render.Renderer(1)
    rng = np.random.default_rng(71)
    srcs = [Source(R1, rng, taps=40, window=("moving", 6000), device="cuda:1"),
            Source(R1, rng, static=True, window=("fixed", 100, 9000), device="cuda:1")]
    s1 = side_stream("cuda:1")
    with torch.cuda.device(0):
        for use_plan in (False, True):
            writes = [w for x in srcs for w in x.writes()]
            outs = [o for x in srcs for o in x.outs()]
            torch.cuda.synchronize(1)
            with torch.cuda.stream(s1):
                for o in outs:
                    o.fill_(NAN)
                for dst, _, p in writes:
                    dst.copy_(p) if isinstance(p, torch.Tensor) else dst.fill_(p)
                torch.cuda._sleep(SLEEP)
                for dst, real, _ in writes:
                    dst.copy_(real)
            assert torch.cuda.current_device() == 0
            with torch.cuda.device(1):
                torch.cuda.set_stream(s1)
            try:
                assert torch.cuda.current_device() == 0
                if use_plan:
                    plan = R1.plan_device([x.py() for x in srcs], [x.out for x in srcs],
                                          direct_outs=[x.dout for x in srcs])
                    plan.run()
                else:
                    R1.render_device([x.py() for x in srcs], [x.out for x in srcs],
                                     direct_outs=[x.dout for x in srcs])
                assert not s1.query()
                with torch.cuda.device(1), torch.cuda.stream(s1):
                    snaps = [o.clone() for o in outs]
            finally:
                with torch.cuda.device(1):
                    torch.cuda.set_stream(torch.cuda.default_stream(1))
            torch.cuda.synchronize(1)
            if use_plan:
                plan.close()
            check_stems(srcs, [c.cpu().numpy() for c in snaps], "cuda:1 %s" % ("plan" if use_plan else "render"))
