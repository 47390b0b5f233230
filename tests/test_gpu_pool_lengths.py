"""Source pools whose candidates differ in L (RIR length) through the real kernels.  Every run writes new picks and
starts, fills the outputs with NaN and runs the plan.  Checked:
  - uniform K, different L (all L <= 4096): aligned speaker pools with a direct target and static noise pools keep
    aligned blocking and k_render_fast (the bits of each candidate rendered alone), and every pooled output and direct stem equals ss_render_dev of the picked candidate with the same
    fixed window, and the slice of its full stem, bit for bit;
  - mixed K (L in {3000, 4097, 9000, 16384}), moving and static, at the first and last start of every candidate: bit
    identity for K_i > 1; for K_i = 1 agreement with the render of its RIRs zero-padded to the pool's longest L within
    float32 rounding (not bit for bit: DESIGN section 3); the float64 per-sample bounds on every output, direct stems
    included;
  - level tables and loudness gains of a mixed-L pool, and the launches of a training plan over it;
  - refusals, ss_pool_bytes and the pool's L;
  - 32 configs[1]-shaped speakers with K = 1..4 in 48 pooled slots with mixtures, against float64."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
import draw_reference as dr
from direct_path import direct_path_rirs
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from draw_reference import Step, TABLE_TOL
from gpu_plumbing import _R
from pool_worlds import Cand, PooledSlots, _draw_training, _training_plan, gain_pool, moving

pytestmark = pytest.mark.gpu

B = 4096
TAPS = 40
NAN = float("nan")


def _k(L):
    return (L + B - 1) // B


def padded(c, L, taps=0):
    """The candidate with its RIRs zero-padded to L taps."""
    h = np.zeros(c.h.shape[:-1] + (L,), np.float32)
    h[..., :c.L] = c.h
    return Cand(c.x, h, c.b, taps)


def static(seed, Ls, N=26000):
    rng = np.random.default_rng(seed)
    return [Cand(so.synth_dry(rng, N + 3001 * j), so.synth_rirs(rng, 1, 2, L)[0], None) for j, L in enumerate(Ls)]


@pytest.mark.parametrize("kind", ["speakers", "noise"])
def test_uniform_k_different_lengths(kind):
    render, R = _R()
    Ls = [1000, 2500, 4096, 1000, 2500]
    cands = moving(40, Ls, TAPS, aligned=1) if kind == "speakers" else static(41, Ls[:3])
    taps = TAPS if kind == "speakers" else 0
    pool = R.source_pool([c.src for c in cands])
    assert pool.L == 4096 and pool.nbytes == 40 * len(cands)
    wl = 9000
    sl = PooledSlots(pool, cands, wl, taps=taps)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    rng = np.random.default_rng(1)
    try:
        for run in range(len(cands) + 4):
            if run < len(cands):                         # the first and last start of every candidate
                p = run
                sl.draw(rng, pk=[p, p, (p + 1) % len(cands), (p + 2) % len(cands), p],
                        st=[0, cands[p].N - wl, 4095, 4097])
            else:
                sl.draw(rng)
            plan.run()
            sl.check("%s run %d" % (kind, run))
        assert plan.is_graph()
        R.check_device_errors()
    finally:
        plan.close()
        pool.close()


def _check_f64(c, y, a, wl, taps, label):
    mode = 0 if c.b is None else 1
    h = direct_path_rirs(c.h, taps) if taps else c.h
    y64, scale = render_check_inputs(c.x, h, mode, bounds=c.b, window=(a, wl))
    check_render(y, y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=a, label=label)


@pytest.mark.parametrize("kind", ["moving", "static"])
def test_mixed_k(kind):
    render, R = _R()
    Ls = [3000, 4097, 9000, 16384]
    taps = TAPS if kind == "moving" else 0
    cands = moving(42, Ls, taps) if kind == "moving" else static(43, Ls)
    pads = {i: padded(c, max(Ls), taps) for i, c in enumerate(cands) if _k(c.L) == 1}
    pool = R.source_pool([c.src for c in cands])
    assert pool.L == 16384 and pool.nbytes == 44 * len(cands)
    wl = 7000
    sl = PooledSlots(pool, cands, wl, taps=taps)
    plan = R.plan_device(sl.srcs, sl.outs, direct_outs=sl.douts)
    n = len(cands)
    try:
        for run in range(n + 2):
            p = run % n
            sl.draw(np.random.default_rng(run), pk=[p, p, (p + 1) % n, (p + 3) % n, (p + 2) % n],
                    st=[0, cands[p].N - wl, cands[(p + 1) % n].N - wl, 0])
            plan.run()
            torch.cuda.synchronize()
            for j, (q, a) in enumerate(zip(sl.pk, sl.st)):
                c = cands[q]
                outs = [(sl.outs[j], c.full, 0)] + ([(sl.douts[j], c.full_d, taps)] if taps else [])
                for k, (y, full, t) in enumerate(outs):
                    what = (kind, run, j, q, a, "direct" if k else "reverberant")
                    if _k(c.L) > 1:
                        assert torch.equal(y, full[:, a:a + wl]), what
                    else:
                        pf = (pads[q].full_d if k else pads[q].full)[:, a:a + wl]
                        err = float((y - pf).abs().max())
                        assert err <= 1e-5 * float(pf.abs().max()), (what, err)
                    _check_f64(c, y.cpu().numpy(), a, wl, t, str(what))
            if run < n:
                ref = [torch.empty_like(o) for o in sl.outs]
                R.render_device([cands[q].src._replace(window=(a, wl)) for q, a in zip(sl.pk, sl.st)], ref)
                torch.cuda.synchronize()
                for j, q in enumerate(sl.pk):
                    if _k(cands[q].L) > 1:
                        assert torch.equal(sl.outs[j], ref[j]), (kind, run, j, q)
        assert plan.is_graph()
        R.check_device_errors()
    finally:
        plan.close()
        pool.close()


def test_levels_gains_and_launches_of_a_mixed_length_pool():
    render, R = _R()
    rng = np.random.default_rng(44)
    spk = []
    for j, L in enumerate([2000, 4096, 6000, 12000, 3000]):
        P, N = 3 + j % 3, 90000 + 7001 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        spk.append(Cand(so.synth_dry(rng, N) * np.float32(0.05 * (j + 1)), so.synth_rirs(rng, P, 2, L), b))
    noi = static(45, [1500, 4096, 5000], N=80000)
    targets = list(rng.uniform(-26, -16, len(spk)))
    sm, nspk = gain_pool(R, render, spk, targets, levels="mono")
    npool = R.source_pool([c.src for c in noi])
    try:
        assert sm.L == 12000 and npool.L == 5000
        assert sm.nbytes == 44 * 5 + 4 * 5 + 8 * sum(c.N + 1 for c in spk) + 8 * 5
        for i, nc in enumerate(nspk):
            # the gain of each candidate measured alone (render_host(..., lufs_targets=))
            assert (sm.loudness[i, 0], sm.loudness[i, 1]) == tuple(nc.loud), i
            q = sm.level_table(i).cpu().numpy()
            ref = dr.level_table(nc.full.cpu().numpy(), True, np.longdouble)
            err = float(np.max(np.abs(q.astype(np.longdouble) - ref)))
            assert err <= TABLE_TOL * float(ref[-1]), (i, err / float(ref[-1]))
        st = Step(R, render, sm, npool, B=4)
        gen = torch.Generator(device="cuda")
        gen.manual_seed(9)
        counts = []
        try:
            for run in range(3):
                st.fill(gen, len(spk), len(noi))
                st.plan.run()
            torch.cuda.synchronize()
            R.reset_stats()
            st.plan.run()
            torch.cuda.synchronize()
            counts.append(R.launch_count())
            assert st.plan.is_graph()
        finally:
            st.plan.close()
        # the same plan over pools whose candidates share one L
        u_spk = R.source_pool([c.src for c in spk[1:2] * 3], levels="mono")
        u_noi = R.source_pool([c.src for c in noi[1:2] * 2])
        st = Step(R, render, u_spk, u_noi, B=4)
        try:
            st.plan.run()
            torch.cuda.synchronize()
            R.reset_stats()
            st.plan.run()
            torch.cuda.synchronize()
            counts.append(R.launch_count())
        finally:
            st.plan.close()
            u_spk.close()
            u_noi.close()
        assert counts[0] == counts[1], counts
        R.check_device_errors()
    finally:
        sm.close()
        npool.close()


def test_refusals_and_sizes():
    from sonicsim_b200 import _lib
    render, R = _R()
    lib = R.lib
    assert lib.ss_version() >= 108
    cands = moving(46, [1000, 9000])
    noi = static(47, [2000])
    rng = np.random.default_rng(0)
    c3 = Cand(so.synth_dry(rng, 30000), so.synth_rirs(rng, 3, 3, 2000), np.array([0, 15000, 30000], np.int32))
    for cs in ([cands[0].src, noi[0].src], [cands[0].src, c3.src]):
        with pytest.raises(ValueError, match="one kind and C"):
            R.source_pool(cs)

    def cand(c, **kw):
        it = _lib.SsSource(x=c.src.dry.data_ptr(), N=c.N, P=len(c.b), C=2, L=c.L, mode=_lib.SS_MOVING_BOUNDS,
                           bounds=c.src.bounds.data_ptr(), bounds_host=c.b.ctypes.data, rir_bank=c.bank._h.value)
        for k, v in kw.items():
            setattr(it, k, v)
        return it

    def create(items):
        arr = (_lib.SsSource * len(items))(*items)
        h = ctypes.c_void_p()
        st = lib.ss_pool_create(R.ctx, arr, len(items), ctypes.byref(h))
        b = lib.ss_pool_bytes(h) if st == 0 else None
        if st == 0:
            lib.ss_pool_destroy(h)
        return st, b

    assert create([cand(cands[0]), cand(cands[1])]) == (0, 88)
    assert create([cand(cands[0]), cand(cands[0])]) == (0, 80)
    assert create([cand(cands[0]), cand(cands[1], L=1000)])[0] == _lib.SS_ERR_INVALID     # not its bank's L
    assert create([cand(cands[0]), cand(c3, C=3)])[0] == _lib.SS_ERR_INVALID
    pool = R.source_pool([c.src for c in cands])
    assert pool.L == 9000 and pool.nbytes == 88
    pick = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.empty((2, 5000), device="cuda")
    d_out = torch.empty((2, 5000), device="cuda")

    def plan(L):
        it = _lib.SsSource(out=d_out.data_ptr(), C=2, L=L, mode=_lib.SS_MOVING_BOUNDS, win_len=5000, pool=pool._h.value,
                           pick_dev=pick.data_ptr())
        p = ctypes.c_void_p()
        st = lib.ss_plan_create(R.ctx, ctypes.byref(it), 1, ctypes.byref(p))
        if st == 0:
            lib.ss_plan_destroy(p)
        return st

    assert plan(9000) == 0
    for L in (1000, 4096, 8999, 9001):
        assert plan(L) == _lib.SS_ERR_INVALID, L
    R.plan_device([render.Pooled(pool, pick, (0, 5000))], [out]).close()
    pool.close()


def test_training_scale_mixed_lengths():
    """32 configs[1]-shaped speakers (C = 6, P = 40) with per-speaker L spread over K = 1..4 and 16 noises; 16 scenes of
    2 pooled speakers and 1 pooled noise (48 pooled slots) with mono mixtures.  Crops of K_i > 1 speakers equal their
    full stems; every sampled crop meets the float64 reference."""
    import bench
    render, R = _R()
    U, S, T = 16, 2, 4 * 16000
    C, N = bench.CFG["C"], bench.CFG["N"]
    items = bench.make_inputs(U, 0)
    rng = np.random.default_rng(18)
    Ls = [1000 + 3997 * (j % 4) + int(rng.integers(0, 3000)) for j in range(2 * U)]    # K = 1, 2, 3, 4
    spk = []
    for j, (x, h, b) in enumerate(items):
        for L in Ls[2 * j:2 * j + 2]:
            hh = np.zeros(h.shape[:-1] + (L,), np.float32)       # configs[1]'s RIRs, cut or given a decaying tail
            hh[..., :min(L, B)] = h[..., :min(L, B)]
            if L > B:
                tail = rng.standard_normal(h.shape[:-1] + (L - B,)) * np.exp(-np.arange(L - B) / 3000.0)
                hh[..., B:] = (tail * 0.01 * float(np.abs(h).max())).astype(np.float32)
            spk.append(Cand(x, hh, b))
    assert {_k(c.L) for c in spk} == {1, 2, 3, 4}
    noi = [Cand((rng.standard_normal(N) * 0.05).astype(np.float32),
                (rng.standard_normal((C, 4096)) * np.exp(-np.arange(4096) / 800.0)).astype(np.float32), None)
           for _ in range(U)]
    sp, np_ = R.source_pool([c.src for c in spk]), R.source_pool([c.src for c in noi])
    assert sp.nbytes == 44 * 2 * U
    plan, st = _training_plan(R, render, sp, np_, U, S, T)
    g = torch.Generator(device="cuda")
    g.manual_seed(6)
    try:
        for run in range(2):
            _draw_training(st, U, S, N, T, g)
            for o in st["outs"]:
                o.fill_(NAN)
            plan.run()
            torch.cuda.synchronize()
            picks, scene, starts = (st[k].cpu().numpy() for k in ("picks", "scene", "starts"))
            for u in range(U):
                a = int(starts[u])
                for k in range(S):
                    c = spk[int(picks[u, k])]
                    y = st["outs"][(S + 1) * u + k]
                    if _k(c.L) > 1:
                        assert torch.equal(y, c.full[:, a:a + T]), (run, u, k)
                    if u in (run, 8 + run):
                        _check_f64(c, y.cpu().numpy(), a, T, 0, "run %d scene %d stem %d" % (run, u, k))
                assert torch.equal(st["outs"][(S + 1) * u + S], noi[int(scene[u])].full[:, a:a + T]), (run, u)
        assert plan.is_graph()
        R.check_device_errors()
    finally:
        plan.close()
        sp.close()
        np_.close()
