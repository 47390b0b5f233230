"""Source pools through the real kernels: pooled slots of device plans (render.Pooled; ss_source.pool + pick_dev) render,
at every run, the candidate a device int32 names.  Every run below draws new picks and starts on the host and writes
them into the plan's tensors on the stream, fills the outputs with NaN and runs the plan.  Checked:
  - every pooled output (and direct-path stem) equals ss_render_dev of the picked candidate with the same fixed window
    at the same start, and the same slice of that candidate's full stem, bit for bit: an aligned speaker pool whose
    candidates differ in P and N, a static noise pool and a long-RIR pool (k_render<LONG>);
  - a pool with mixed blocking renders every candidate on the grid, within the float64 bounds of DESIGN section 5;
  - one candidate picked by two slots, one pool in many slots and two live plans, a pool closed under a live plan;
  - mixtures over pooled slots equal ss_mix_dev on the picked crops;
  - picks and starts out of range are clamped and reported (IndexError / ValueError);
  - the graph, and launches per run equal to a plan of the same slots as fixed banked moving-window sources;
  - every refusal, in Python and through the C ABI;
  - bench.py's 16 configs[1] utterances as a pool of 32 speakers and 16 noises, 48 pooled slots with mixtures."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from gpu_plumbing import _R, to
from pool_worlds import (Cand, PooledSlots, TAPS, _draw_training, _mix_dev, _training_plan, fold_dev, longs, noises,
                         speakers)
from window_cases import _choice

pytestmark = pytest.mark.gpu

NAN = float("nan")


def mixed(seed):
    """Two candidates that would choose aligned blocking and two that would choose the grid (many short segments)."""
    rng = np.random.default_rng(seed)
    out = speakers(seed, n=2, taps=0)
    for j in range(2):
        P, N = 40, 20000 + 3000 * j
        np.random.seed(seed + j)
        idx, _ = so.setup_dynamic_interp(so.synth_path(rng, P), N)
        b = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)
        assert _choice(b, N, P, 4096) == 0
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    return out


POOLS = {"speakers": speakers, "noise": noises, "long": longs}


@pytest.mark.parametrize("kind", list(POOLS))
def test_pooled_outputs_equal_the_picked_candidate(kind):
    render, R = _R()
    cands = POOLS[kind](7)
    pool = R.source_pool([c.src for c in cands])
    taps = TAPS if kind == "speakers" else 0
    wl = 9000
    sl = PooledSlots(pool, cands, wl, taps=taps)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    rng = np.random.default_rng(1)
    try:
        for run in range(20):
            if run == 0:                    # one candidate in two slots; the first and last start of its range
                p = len(cands) - 1
                sl.draw(rng, pk=[p, p, 0, 1, 2], st=[0, cands[p].N - wl, 4095, 4097])
            else:
                sl.draw(rng)
            plan.run()
            sl.check("%s run %d" % (kind, run))
        assert plan.is_graph()
        R.check_device_errors()
    finally:
        plan.close()
        pool.close()


def test_launches_equal_fixed_moving_windows():
    """A pooled plan runs as one graph with the launches of a plan of the same slots as fixed banked moving windows."""
    render, R = _R()
    cands = speakers(8, taps=0)
    pool = R.source_pool([c.src for c in cands])
    sl = PooledSlots(pool, cands, 9000)
    fixed = [c.src._replace(window=(sl.starts[j], 9000)) for j, c in enumerate(cands[:4])]
    fixed.append(cands[4].src._replace(window=(sl.fixed, 9000)))
    p_pool = R.plan_device(sl.srcs, sl.outs)
    p_fix = R.plan_device(fixed, [torch.empty_like(o) for o in sl.outs])
    try:
        counts = []
        for plan in (p_pool, p_fix):
            plan.run()
            c0 = R.launch_count()
            plan.run()
            plan.run()
            counts.append((R.launch_count() - c0) // 2)
            assert plan.is_graph()
        assert counts[0] == counts[1] and counts[0] % 3 == 0, counts
    finally:
        p_pool.close()
        p_fix.close()
        pool.close()


def test_mixed_blocking_against_float64():
    """Aligned-eligible candidates in a pool with grid-choosing ones render on the grid: per-sample bounds against
    the float64 reference."""
    render, R = _R()
    cands = mixed(9)
    pool = R.source_pool([c.src for c in cands])
    wl = 12000
    sl = PooledSlots(pool, cands, wl)
    plan = R.plan_device(sl.srcs, sl.outs)
    rng = np.random.default_rng(2)
    try:
        seen = set()
        for run in range(6):
            sl.draw(rng, pk=[run % 4, (run + 1) % 4, (run + 2) % 4, (run + 3) % 4, run % 4])
            plan.run()
            torch.cuda.synchronize()
            for j, (p, a) in enumerate(zip(sl.pk, sl.st)):
                c = cands[p]
                y = sl.outs[j].cpu().numpy()
                y64, scale = render_check_inputs(c.x, c.h, 1, bounds=c.b, window=(a, wl))
                check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=a, label="run %d slot %d cand %d" % (run, j, p))
                seen.add(p)
        assert seen == set(range(4))
        R.check_device_errors()
    finally:
        plan.close()
        pool.close()


def test_pool_shared_by_plans_and_closed_under_them():
    render, R = _R()
    cands = noises(10)
    pool = R.source_pool([c.src for c in cands])
    assert pool.nbytes == 40 * len(cands)
    a, b = PooledSlots(pool, cands, 5000), PooledSlots(pool, cands, 7000, k=6)
    pa, pb = R.plan_device(a.srcs, a.outs), R.plan_device(b.srcs, b.outs)
    pool.close()                                          # both plans keep it alive
    assert pool.closed and pool._h
    with pytest.raises(ValueError, match="closed"):
        R.plan_device(a.srcs, a.outs)
    rng = np.random.default_rng(3)
    try:
        for run in range(4):
            a.draw(rng)
            b.draw(rng)
            pa.run()
            pb.run()
            a.check("plan a run %d" % run)
            b.check("plan b run %d" % run)
        pa.close()
        assert pool._h
        b.draw(rng)
        pb.run()
        b.check("plan b alone")
    finally:
        pa.close()
        pb.close()
    assert not pool._h                                    # freed with the last plan


def _check_training(R, st, spk_cands, noi_cands, S, T, what):
    """Every crop is the slice of its picked candidate's full stem; every mixture equals ss_mix_dev on the crops."""
    torch.cuda.synchronize()
    picks, scene, starts = (st[k].cpu().numpy() for k in ("picks", "scene", "starts"))
    U = len(scene)
    for u in range(U):
        a = int(starts[u])
        crops = []
        for k in range(S + 1):
            c = spk_cands[int(picks[u, k])] if k < S else noi_cands[int(scene[u])]
            o = st["outs"][(S + 1) * u + k]
            assert torch.equal(o, c.full[:, a:a + T]), (what, u, k, a)
            crops.append(fold_dev(o))
        mix, out = _mix_dev(R, torch.stack(crops[:S]), torch.stack(crops[S:]), st["sirs"][u], st["snr"][u])
        assert torch.equal(mix, st["mix"][u]) and torch.equal(out, st["spk_out"][u]), (what, u)


def test_mixtures_over_pooled_slots():
    render, R = _R()
    S, T, n_scenes = 2, 8000, 3
    spk = speakers(11, n=S * n_scenes, taps=0)
    noi = noises(12, n=n_scenes)
    sp, np_ = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])
    plan, st = _training_plan(R, render, sp, np_, 4, S, T)
    g = torch.Generator(device="cuda")
    g.manual_seed(4)
    try:
        for run in range(5):
            _draw_training(st, n_scenes, S, min(sp.n_min, np_.n_min), T, g)
            plan.run()
            _check_training(R, st, spk, noi, S, T, "run %d" % run)
        R.check_device_errors()
    finally:
        plan.close()
        sp.close()
        np_.close()


def test_out_of_range_picks_and_starts_are_clamped():
    render, R = _R()
    cands = noises(13)
    pool = R.source_pool([c.src for c in cands])
    wl = 6000
    sl = PooledSlots(pool, cands, wl, k=2)
    plan = R.plan_device(sl.srcs, sl.outs)
    n = len(cands)
    try:
        R.check_device_errors()
        # picks outside [0, n): the last / first candidate, IndexError
        sl.draw(None, pk=[n + 5, -3, n], st=[10, 20])
        plan.run()
        sl.pk = [n - 1, 0, n - 1]
        sl.check("clamped picks")
        with pytest.raises(IndexError):
            R.check_device_errors()
        R.check_device_errors()
        # a start past the picked candidate's N - wl (it is within the longest candidate's): clamped, ValueError
        short = 0
        sl.draw(None, pk=[short, n - 1, 1], st=[cands[short].N - wl + 7, cands[n - 1].N - wl])
        plan.run()
        sl.st[0] = cands[short].N - wl
        sl.check("clamped start")
        with pytest.raises(ValueError):
            R.check_device_errors()
    finally:
        plan.close()
        pool.close()


def test_python_refusals():
    render, R = _R()
    cands = speakers(14, n=2, taps=0)
    noi = noises(15, n=2)
    good = [c.src for c in cands]
    rng = np.random.default_rng(0)
    raw = render.MovingSource(to(cands[0].x), to(cands[0].h), to(cands[0].b), cands[0].b)
    bad_pools = {
        "empty": [],
        "raw RIRs": [raw],
        "window": [good[0]._replace(window=(0, 10))],
        "normalize": [good[0]._replace(normalize_rirs=True)],
        "direct_taps": [good[0]._replace(direct_taps=TAPS)],
        "no bounds_host": [good[0]._replace(bounds_host=None)],
        "host dry": [good[0]._replace(dry=cands[0].x)],
        "int64 bounds": [good[0]._replace(bounds=to(cands[0].b.astype(np.int64)))],
        "mixed kinds": [good[0], noi[0].src],
        "mixed C": [good[0], Cand(so.synth_dry(rng, 30000), so.synth_rirs(rng, 3, 3, 4096),
                                  np.array([0, 15000, 30000], np.int32)).src],
        "not a source": [good[0], 5],
    }
    for what, cs in bad_pools.items():
        with pytest.raises(ValueError):
            R.source_pool(cs)
        assert what
    pool = R.source_pool(good)
    npool = R.source_pool([c.src for c in noi])
    pick = torch.zeros(1, dtype=torch.int32, device="cuda")
    wl = 5000
    out = torch.empty((2, wl), device="cuda")
    ok = render.Pooled(pool, pick, (0, wl))
    R.plan_device([ok], [out]).close()
    bad_slots = {
        "no window": (ok._replace(window=None), None),
        "window too long": (ok._replace(window=(0, pool.n_min + 1)), None),
        "fixed start too late": (ok._replace(window=(pool.n_min - wl + 1, wl)), None),
        "int64 pick": (ok._replace(pick=torch.zeros(1, dtype=torch.int64, device="cuda")), None),
        "two picks": (ok._replace(pick=torch.zeros(2, dtype=torch.int32, device="cuda")), None),
        "host pick": (ok._replace(pick=torch.zeros(1, dtype=torch.int32)), None),
        "not a pool": (ok._replace(pool=cands[0].bank), None),
        "direct without a direct set": (render.Pooled(npool, pick, (0, wl), TAPS), [out.clone()]),
        "direct without an output": (ok._replace(direct_taps=TAPS), None),
        "wrong output shape": (ok._replace(window=(0, wl - 1)), None),
    }
    for what, (s, douts) in bad_slots.items():
        with pytest.raises(ValueError):
            R.plan_device([s], [out], direct_outs=douts)
        assert what
    with pytest.raises(ValueError, match="pooled"):
        R.render_device([ok], [out])
    with pytest.raises(ValueError, match="pooled"):
        R.render_host([ok])
    with pytest.raises(ValueError, match="pooled"):
        R.plan_host([ok])
    npool.close()
    with pytest.raises(ValueError, match="closed"):
        R.plan_device([render.Pooled(npool, pick, (0, wl))], [out])
    pool.close()


def test_c_abi_refusals():
    from sonicsim_b200 import _lib
    render, R = _R()
    lib = R.lib
    cands = speakers(16, n=2, taps=0)
    c0 = cands[0]
    d_out = torch.empty((2, 5000), device="cuda")
    d_pick = torch.zeros(2, dtype=torch.int32, device="cuda")

    def cand(**kw):
        it = _lib.SsSource(x=c0.src.dry.data_ptr(), N=c0.N, P=len(c0.b), C=2, L=4096, mode=_lib.SS_MOVING_BOUNDS,
                           bounds=c0.src.bounds.data_ptr(), bounds_host=c0.b.ctypes.data, rir_bank=c0.bank._h.value)
        for k, v in kw.items():
            setattr(it, k, v)
        return it

    def create(items):
        arr = (_lib.SsSource * len(items))(*items)
        h = ctypes.c_void_p()
        st = lib.ss_pool_create(R.ctx, arr, len(items), ctypes.byref(h))
        if st == 0:
            lib.ss_pool_destroy(h)
        return st

    assert create([cand()]) == 0
    d_h = to(c0.h)
    for kw in [dict(rir=d_h.data_ptr(), rir_bank=None), dict(rir_bank=None), dict(mode=_lib.SS_MOVING_INDEXED),
               dict(bounds_host=None), dict(out=d_out.data_ptr()), dict(win_len=100), dict(flags=_lib.SS_DIRECT_TARGET),
               dict(L=4097), dict(P=2), dict(x=None), dict(pick_dev=d_pick.data_ptr()), dict(mode=_lib.SS_STATIC)]:
        assert create([cand(**kw)]) == _lib.SS_ERR_INVALID, kw
    assert create([cand(), cand(C=3)]) == _lib.SS_ERR_INVALID
    h = ctypes.c_void_p()
    assert lib.ss_pool_create(R.ctx, (_lib.SsSource * 1)(cand()), 0, ctypes.byref(h)) == _lib.SS_ERR_INVALID
    pool = R.source_pool([c.src for c in cands])

    def slot(**kw):
        it = _lib.SsSource(out=d_out.data_ptr(), C=2, L=4096, mode=_lib.SS_MOVING_BOUNDS, win_len=5000,
                           pool=pool._h.value, pick_dev=d_pick.data_ptr())
        for k, v in kw.items():
            setattr(it, k, v)
        return it

    def plan(it):
        p = ctypes.c_void_p()
        st = lib.ss_plan_create(R.ctx, ctypes.byref(it), 1, ctypes.byref(p))
        if st == 0:
            lib.ss_plan_destroy(p)
        return st

    assert plan(slot()) == 0
    assert plan(slot(win_start_dev=d_pick.data_ptr() + 4)) == 0
    for kw in [dict(x=c0.src.dry.data_ptr()), dict(N=c0.N), dict(P=3), dict(rir_bank=c0.bank._h.value),
               dict(bounds=c0.src.bounds.data_ptr()), dict(mode=_lib.SS_STATIC), dict(C=1), dict(L=300),
               dict(win_len=0), dict(win_len=pool.n_min + 1), dict(win_start=pool.n_min - 4999),
               dict(flags=_lib.SS_RIR_NORMALIZE), dict(pick_dev=d_pick.data_ptr() + 2), dict(pick_dev=None),
               dict(out=None), dict(win_start_dev=d_pick.data_ptr() + 2),
               dict(flags=_lib.SS_DIRECT_TARGET, out_direct=d_out.data_ptr() + 4, direct_taps=TAPS)]:
        assert plan(slot(**kw)) == _lib.SS_ERR_INVALID, kw
    it = slot()
    stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    assert lib.ss_render_dev(R.ctx, ctypes.byref(it), 1, stream) == _lib.SS_ERR_INVALID
    assert lib.ss_render_host(R.ctx, ctypes.byref(it), 1) == _lib.SS_ERR_INVALID
    assert lib.ss_render_host_ex(R.ctx, ctypes.byref(it), 1, None) == _lib.SS_ERR_INVALID
    pool.close()


def test_training_scale_pool():
    """bench.py's 16 configs[1] utterances as a pool of 32 banked speakers and 16 banked noises; 16 scenes of 2 pooled
    speakers and 1 pooled noise each (48 pooled slots) with mono mixtures; crops equal the picked candidates' full stems
    and sampled crops meet the float64 reference."""
    import bench
    render, R = _R()
    U, S, T = 16, 2, 4 * 16000
    C, N = bench.CFG["C"], bench.CFG["N"]
    items = bench.make_inputs(U, 0)
    rng = np.random.default_rng(17)
    spk = [Cand(x, h, b) for x, h, b in items]
    noi = [Cand((rng.standard_normal(N) * 0.05).astype(np.float32),
                (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32), None)
           for _ in range(U)]
    sp, np_ = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])
    plan, st = _training_plan(R, render, sp, np_, U, S, T)
    g = torch.Generator(device="cuda")
    g.manual_seed(5)
    try:
        for run in range(3):
            _draw_training(st, U, S, N, T, g)
            plan.run()
            _check_training(R, st, spk, noi, S, T, "run %d" % run)
        picks, scene, starts = (st[k].cpu().numpy() for k in ("picks", "scene", "starts"))
        for u in (0, 7, 15):
            a = int(starts[u])
            for k in range(S + 1):
                c = spk[int(picks[u, k])] if k < S else noi[int(scene[u])]
                y = st["outs"][(S + 1) * u + k].cpu().numpy()
                y64, scale = render_check_inputs(c.x, c.h, 1 if c.b is not None else 0, bounds=c.b, window=(a, T))
                check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=a, label="scene %d stem %d" % (u, k))
        assert plan.is_graph()
        R.check_device_errors()
    finally:
        plan.close()
        sp.close()
        np_.close()
