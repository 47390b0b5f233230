"""Host pools (SS_BANK_HOST, Renderer.rir_bank(host=True)) through the real kernels: every candidate's bank, dry signal and
level table in pinned host memory, and k_stage copying each run's read sets to the device.  Checked:
  1. banks: a host bank holds no device memory, host_nbytes follows 8 * 4096 * P * C * K per set plus the cut table, and
     a whole-stem slot over it (every row and sample staged) equals render_device over the device bank, bit for bit;
  2. bit identity: one training plan - pooled speakers with direct targets in a mixed-L pool with loudness gains, static
     noise and music pools, CropDraws, Mixtures with mono and noise_delay - built over device pools and over host pools
     of the same candidates gives the same stems, direct stems, mixes, speakers_out, rms_db, drawn starts and `used` over
     22 runs with new picks, u, SIRs and SNRs; probe slots take every candidate's first and last start, and one run an
     out-of-range pick and start, which check_device_errors reports alike; level tables and loudness are equal;
  3. device memory: building a host pool with level tables over 283 MB of banks grows device memory by at most 32 MB
     (ss_pool_bytes plus driver pages), and ss_pool_bytes is 40 n + 4 sum(P) + 8 n (entries, bounds, level table
     pointers);
  4. launches: a run of the host-pool plan launches one kernel more than the device-pool plan, as one graph launch;
  5. a side stream gives the same bits;
  6. refusals of host banks outside host pools and of pools that mix host and device banks, in Python and the C ABI.
The tests hold well under 2 GB of pinned host memory."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from gpu_plumbing import _R, _errors, to

pytestmark = pytest.mark.gpu

RATE = 16000
LEN = 2 * RATE
TRIES = 101
TAPS = 40


class Cand:
    def __init__(self, rng, N, P, C, L):
        self.x = so.synth_dry(rng, N)
        self.x[int(rng.integers(0, N // 2)):][:int(rng.integers(0, N // 3))] = 0      # a silent stretch
        self.h = so.synth_rirs(rng, P, C, L)
        self.b = None if P == 1 else np.round(np.linspace(0, N, P)).astype(np.int32)
        self.N, self.P, self.C, self.L = N, P, C, L


def _pool(R, render, cands, host, taps=0, levels=None, lufs=None):
    out = []
    for c in cands:
        bank = R.rir_bank(c.h if c.P > 1 else c.h[0], direct_taps=taps, host=host)
        if c.P == 1:
            out.append(render.StaticSource(c.x if host else to(c.x), bank))
        elif host:                                   # NumPy dry and bounds: the pool copies them
            out.append(render.MovingSource(c.x, bank, c.b))
        else:
            out.append(render.MovingSource(to(c.x), bank, to(c.b), bounds_host=c.b))
    return R.source_pool(out, levels=levels, lufs_targets=lufs, sr=RATE)


@pytest.fixture(scope="module")
def world():
    render, R = _R()
    rng = np.random.default_rng(2026)
    spk = [Cand(rng, 120000 + 9001 * j, 3 + j % 4, 2, (4096, 9000, 3000)[j % 3]) for j in range(7)]
    noi = [Cand(rng, 100000 + 13007 * j, 1, 2, (4096, 6000)[j % 2]) for j in range(4)]
    mus = [Cand(rng, 90000 + 7919 * j, 1, 2, 2048) for j in range(3)]
    pools = {}
    for host in (False, True):
        pools[host] = (
            _pool(R, render, spk, host, TAPS, "mono", [-17.0 + 0.5 * j for j in range(len(spk))]),
            _pool(R, render, noi, host, 0, None, [-24.0, None, -23.0, -25.0]),
            _pool(R, render, mus, host, 0, None, None))
    return spk, noi, mus, pools


B = 3                                               # examples; each: 2 speakers, noise, music + 3 probe slots


class Inputs:
    def __init__(self):
        self.picks = torch.zeros((B, 4), dtype=torch.int32, device="cuda")
        self.probe_pick = torch.zeros(3, dtype=torch.int32, device="cuda")
        self.probe_start = torch.zeros(3, dtype=torch.int32, device="cuda")
        self.u = torch.zeros((B, TRIES), dtype=torch.float64, device="cuda")
        self.sirs = torch.zeros((B, 1), device="cuda")
        self.snr = torch.zeros((B, 1), device="cuda")


def _plan(render, R, pools, inp):
    spk, noi, mus = pools
    starts = torch.zeros(B, dtype=torch.int32, device="cuda")
    used = torch.zeros(B, dtype=torch.int32, device="cuda")
    o = {"out": [], "direct": [], "mix": [], "spk_out": [], "rms": [], "starts": starts, "used": used}
    sources, direct_outs, mixtures, draws = [], [], [], []
    for b in range(B):
        base = len(sources)
        for k, pl in enumerate((spk, spk, noi, mus)):
            taps = TAPS if k < 2 else 0
            sources.append(render.Pooled(pl, inp.picks[b, k], (starts[b], LEN), taps))
            o["out"].append(torch.zeros((2, LEN), device="cuda"))
            direct_outs.append(torch.zeros((2, LEN), device="cuda") if taps else None)
        mono = b % 2 == 0
        shape = (LEN,) if mono else (2, LEN)
        o["mix"].append(torch.zeros(shape, device="cuda"))
        o["spk_out"].append(torch.zeros((2,) + shape, device="cuda"))
        o["rms"].append(torch.zeros(2, device="cuda"))
        mixtures.append(render.Mixture([base, base + 1], [base + 2, base + 3], inp.sirs[b], inp.snr[b], o["mix"][-1],
                                       o["spk_out"][-1], o["rms"][-1], mono, 0 if b == 1 else 3))
        draws.append(render.CropDraw(starts[b], [base, base + 1], inp.u[b], used[b]))
    for k, pl in enumerate((spk, noi, mus)):      # probes: starts written by the host, any candidate, any start
        sources.append(render.Pooled(pl, inp.probe_pick[k], (inp.probe_start[k], LEN), TAPS if k == 0 else 0))
        o["out"].append(torch.zeros((2, LEN), device="cuda"))
        direct_outs.append(torch.zeros((2, LEN), device="cuda") if k == 0 else None)
    o["direct"] = [d for d in direct_outs if d is not None]
    plan = R.plan_device(sources, o["out"], direct_outs=direct_outs, mixtures=mixtures, draws=draws)
    return plan, o


def _same(a, b, what):
    for k in ("out", "direct", "mix", "spk_out", "rms"):
        for i, (x, y) in enumerate(zip(a[k], b[k])):
            assert torch.equal(x, y), (what, k, i)
    assert torch.equal(a["starts"], b["starts"]) and torch.equal(a["used"], b["used"]), what


def test_pools_and_builds_equal(world):
    spk, noi, mus, pools = world
    for d, h in zip(pools[False], pools[True]):
        assert d.resident == "device" and h.resident == "host"
        assert np.array_equal(d.loudness, h.loudness, equal_nan=True)
        assert h.host_nbytes > 0 and d.host_nbytes == 0
    d, h = pools[False][0], pools[True][0]
    for i in range(d.n):
        assert torch.equal(d.level_table(i), h.level_table(i)), i


def test_training_plan_bit_identity(world):
    render, R = _R()
    spk, noi, mus, pools = world
    inp = Inputs()
    pd, od = _plan(render, R, pools[False], inp)
    ph, oh = _plan(render, R, pools[True], inp)
    rng = np.random.default_rng(7)
    counts = (len(spk), len(spk), len(noi), len(mus))
    probes = [[(i, s) for i, c in enumerate(cs) for s in (0, c.N - LEN)] for cs in (spk, noi, mus)]
    runs = max(22, max(len(q) for q in probes) + 2)
    R.check_device_errors()
    for r in range(runs):
        picks = np.array([[rng.integers(0, n) for n in counts] for _ in range(B)], np.int32)
        inp.picks.copy_(torch.from_numpy(picks))
        u = rng.random((B, TRIES))
        if r % 5 == 1:
            u[:] = 0.0                               # the first start
        elif r % 5 == 2:
            u[:] = 1.0                               # the last start of the shortest reader
        inp.u.copy_(torch.from_numpy(u))
        inp.sirs.uniform_(-6, 6)
        inp.snr.uniform_(10, 20)
        pp, ps = np.zeros(3, np.int32), np.zeros(3, np.int32)
        for k in range(3):                           # every candidate's first and last start, then the middle
            pp[k], ps[k] = probes[k].pop(0) if probes[k] else (r % counts[k + (k > 0)], LEN // 3)
        bad = r == runs - 1
        if bad:                                      # out of range: clamped, and reported alike
            pp[:] = [len(spk) + 3, -2, 99]
            ps[:] = [-5, 10 ** 7, 3]
        inp.probe_pick.copy_(torch.from_numpy(pp))
        inp.probe_start.copy_(torch.from_numpy(ps))
        pd.run()
        ed = _errors(R)
        ph.run()
        eh = _errors(R)
        assert ed == eh, (r, ed, eh)
        assert (ed is not None) == bad, (r, ed)
        _same(od, oh, r)
    assert not any(probes)
    assert pd.is_graph() and ph.is_graph()


def test_launches_and_side_stream(world):
    render, R = _R()
    spk, noi, mus, pools = world
    inp = Inputs()
    pd, od = _plan(render, R, pools[False], inp)
    ph, oh = _plan(render, R, pools[True], inp)
    inp.picks.copy_(torch.tensor([[1, 2, 3, 0], [4, 6, 1, 2], [0, 5, 2, 1]], dtype=torch.int32))
    inp.u.uniform_()
    inp.sirs.fill_(2.5)
    inp.snr.fill_(15.0)
    inp.probe_pick.fill_(1)
    inp.probe_start.fill_(777)
    pd.run(); ph.run()                               # graphs captured
    torch.cuda.synchronize()
    n = []
    for p in (pd, ph):
        R.reset_stats()
        p.run()
        n.append(R.launch_count())
    assert n[1] == n[0] + 1, n
    assert pd.is_graph() and ph.is_graph()
    torch.cuda.synchronize()
    ref = {k: [t.clone() for t in v] if isinstance(v, list) else v.clone() for k, v in oh.items()}
    for v in oh.values():
        for t in (v if isinstance(v, list) else [v]):
            t.fill_(-1)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        torch.cuda._sleep(int(2e7))                  # queued work in front of the run
        ph.run(s.cuda_stream)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    _same(ref, oh, "side stream")
    _same(od, oh, "against the device pools")


def test_host_bank_and_whole_stem(world):
    render, R = _R()
    rng = np.random.default_rng(3)
    c = Cand(rng, 50000, 5, 3, 9000)
    hb = R.rir_bank(c.h, direct_taps=TAPS, host=True)
    db = R.rir_bank(c.h, direct_taps=TAPS)
    K = (c.L + 4095) // 4096
    assert hb.host and not db.host and hb.nbytes == 0 and db.host_nbytes == 0
    assert hb.host_nbytes == 2 * 8 * 4096 * c.P * c.C * K + 4 * c.P * c.C
    ref, ref_d = torch.zeros((3, c.N), device="cuda"), torch.zeros((3, c.N), device="cuda")
    R.render_device([render.MovingSource(to(c.x), db, to(c.b), bounds_host=c.b, direct_taps=TAPS)], [ref],
                    direct_outs=[ref_d])
    pool = R.source_pool([render.MovingSource(c.x, hb, c.b)])
    pick, y, yd = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros_like(ref), torch.zeros_like(ref)
    plan = R.plan_device([render.Pooled(pool, pick[0], (0, c.N), TAPS)], [y], direct_outs=[yd])
    plan.run()
    torch.cuda.synchronize()
    assert torch.equal(y, ref) and torch.equal(yd, ref_d)


def test_device_memory_of_a_host_pool():
    render, R = _R()
    rng = np.random.default_rng(11)
    n, P, C, N = 24, 60, 6, 30 * RATE
    b = np.round(np.linspace(0, N, P)).astype(np.int32)
    h = so.synth_rirs(rng, P, C, 4096)
    x = so.synth_dry(rng, N)
    banks = [R.rir_bank(h, host=True) for _ in range(n)]
    assert sum(k.host_nbytes for k in banks) == n * 8 * 4096 * P * C
    cands = [render.MovingSource(x, banks[i], b) for i in range(n)]
    R.source_pool(cands, levels="channels").close()   # the context's own render scratch grows to this build's size
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    pool = R.source_pool(cands, levels="channels")
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    grown = free0 - torch.cuda.mem_get_info()[0]
    assert pool.nbytes == 40 * n + 4 * n * P + 8 * n, pool.nbytes
    # the build's transient buffers are freed; what stays besides the pool is a few MB of driver pages (19.8 MB
    # measured on an H100 80GB HBM3), against 283 MB of banks and 138 MB of dry signals and tables on the host
    assert grown <= pool.nbytes + (32 << 20), (grown, pool.nbytes)
    assert pool.host_nbytes == n * (4 * N + 8 * (N + 1)), pool.host_nbytes
    pool.close()
    for k in banks:
        k.close()


def test_refusals(world):
    render, R = _R()
    lib = R.lib
    from sonicsim_b200 import _lib
    rng = np.random.default_rng(5)
    c = Cand(rng, 20000, 3, 2, 4096)
    hb, db = R.rir_bank(c.h, host=True), R.rir_bank(c.h)
    src = render.MovingSource(to(c.x), hb, to(c.b), bounds_host=c.b)
    out = torch.zeros((2, c.N), device="cuda")
    with pytest.raises(ValueError, match="host bank"):
        R.render_device([src], [out])
    with pytest.raises(ValueError, match="host bank"):
        R.plan_device([src], [out])
    with pytest.raises(ValueError, match="host bank"):
        R.render_host([render.MovingSource(c.x, hb, c.b)])
    with pytest.raises(ValueError, match="host bank"):
        R.plan_host([render.MovingSource(c.x, hb, c.b)])
    with pytest.raises(ValueError, match="host banks or all device banks"):
        R.source_pool([render.MovingSource(to(c.x), db, to(c.b), bounds_host=c.b), render.MovingSource(c.x, hb, c.b)])
    # the C ABI
    item = _lib.SsSource(x=src.dry.data_ptr(), out=out.data_ptr(), bounds=src.bounds.data_ptr(),
                         bounds_host=c.b.ctypes.data, N=c.N, P=c.P, C=2, L=c.L, mode=_lib.SS_MOVING_BOUNDS,
                         rir_bank=hb._h.value)
    assert lib.ss_render_dev(R.ctx, ctypes.byref(item), 1, None) == _lib.SS_ERR_INVALID
    h = ctypes.c_void_p()
    assert lib.ss_plan_create(R.ctx, ctypes.byref(item), 1, ctypes.byref(h)) == _lib.SS_ERR_INVALID and not h.value
    hitem = _lib.SsSource(x=c.x.ctypes.data, out=np.zeros((2, c.N), np.float32).ctypes.data, bounds=c.b.ctypes.data,
                          N=c.N, P=c.P, C=2, L=c.L, mode=_lib.SS_MOVING_BOUNDS, rir_bank=hb._h.value)
    assert lib.ss_render_host(R.ctx, ctypes.byref(hitem), 1) == _lib.SS_ERR_INVALID
    cand = (_lib.SsSource * 2)()
    for i, bank in enumerate((db, hb)):
        cand[i] = _lib.SsSource(x=src.dry.data_ptr(), bounds=src.bounds.data_ptr(), bounds_host=c.b.ctypes.data, N=c.N,
                                P=c.P, C=2, L=c.L, mode=_lib.SS_MOVING_BOUNDS, rir_bank=bank._h.value)
    assert lib.ss_pool_create(R.ctx, cand, 2, ctypes.byref(h)) == _lib.SS_ERR_INVALID and not h.value
    # a host pool's candidate needs no device bounds
    cand[0] = cand[1]
    cand[0].bounds = None
    assert lib.ss_pool_create(R.ctx, cand, 1, ctypes.byref(h)) == _lib.SS_OK
    lib.ss_pool_destroy(h)
    hb.close()
    db.close()
