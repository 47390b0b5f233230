"""Start draws of device plans (render.CropDraw; ss_plan_draw) and level tables of pools (ss_pool_levels) through the real
kernels.  The dry signals have create_long_audio-style gaps (0-10 s of silence before every burst of speech) and the
candidates differ in N, so many 4 s crops are silent.  Checked:
  1. tables: mono and channel tables of a moving and a static pool against the float64 prefix sums of ss_render_dev's
     whole stems (a long-double reference; bound TABLE_TOL * Q[N]), and two builds give identical bits;
  2. draws: over many runs with new u and picks written on the device and no host synchronisation, every start and
     `used` equals tests/draw_reference.py on the device's own tables (draws whose levels lie within NEAR_DB of the
     threshold are left out, and must be rare); every stem equals the picked candidate's full ss_render_dev stem at the
     drawn start, bit for bit; rms_db >= threshold - 1e-5 wherever a try was accepted; no error bit (no start or pick was
     clamped), also when the shortest reader is a noise and u = 1 maps to its last start;
  3. all silent: used == 0 and the last try's start;
  4. launches: a run with draws launches one kernel more than the same plan without; the no-graph and profiling paths
     give the same bits;
  5. a side stream behind queued work, with u and the picks written on it;
  6. every refusal, in Python and through the C ABI, with nothing written."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
import draw_reference as dr
from draw_reference import LEN, Step, TABLE_TOL, check_snap, gappy_dry
from gpu_plumbing import _R, to
from pool_worlds import Cand
from window_cases import _choice

pytestmark = pytest.mark.gpu

NAN = float("nan")
SLEEP = int(5e8)


@pytest.fixture(scope="module")
def world():
    rng = np.random.default_rng(107)
    spk, noi = [], []
    for j in range(6):                                   # moving speakers, aligned blocking, N from 12.5 s to 24 s
        P, N = 3 + j % 3, 200000 + 37003 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        assert _choice(b, N, P, 4096) == 1
        spk.append(Cand(gappy_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    for j in range(4):                                   # static noises, the shortest shorter than every speaker
        noi.append(Cand(so.synth_dry(rng, 150000 + 97001 * j), so.synth_rirs(rng, 1, 2, 4096)[0], None))
    return spk, noi


def tables(pool):
    return [pool.level_table(i).cpu().numpy() for i in range(pool.n)]


@pytest.mark.parametrize("kind", ["moving", "static"])
def test_level_tables(world, kind):
    render, R = _R()
    cands = world[0] if kind == "moving" else world[1]
    n = len(cands)
    plain = R.source_pool([c.src for c in cands])
    assert plain.levels is None and plain.nbytes == 40 * n and plain.level_table(0) is None
    plain.close()
    for levels in ("mono", "channels"):
        a = R.source_pool([c.src for c in cands], levels=levels)
        b = R.source_pool([c.src for c in cands], levels=levels)
        try:
            assert a.levels == levels
            assert a.nbytes == 40 * n + 8 * sum(c.N + 1 for c in cands) + 8 * n
            for i, c in enumerate(cands):
                q, q2 = a.level_table(i), b.level_table(i)
                assert torch.equal(q, q2), (kind, levels, i)
                ref = dr.level_table(c.full.cpu().numpy(), levels == "mono", np.longdouble)
                qn = q.cpu().numpy()
                assert qn.shape == (c.N + 1,) and qn[0] == 0.0
                err = float(np.max(np.abs(qn.astype(np.longdouble) - ref)))
                assert err <= TABLE_TOL * float(ref[-1]), (kind, levels, i, err / float(ref[-1]))
        finally:
            a.close()
            b.close()


@pytest.fixture(scope="module")
def pools(world):
    _, R = _R()
    spk, noi = world
    sm = R.source_pool([c.src for c in spk], levels="mono")
    sc = R.source_pool([c.src for c in spk], levels="channels")
    npool = R.source_pool([c.src for c in noi])
    yield sm, sc, npool, tables(sm), tables(sc)
    for p in (sm, sc, npool):
        p.close()


def test_draws_equal_the_reference(world, pools):
    render, R = _R()
    spk, noi = world
    sm, _, npool, Tm, _ = pools
    st = Step(R, render, sm, npool, B=16)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(11)
    snaps = []
    longest = torch.tensor([4, 5, 0], dtype=torch.int32, device="cuda")
    try:
        for run in range(10):
            st.fill(gen, len(spk), len(noi))
            if run == 0:
                # example 0: the two longest speakers over the shortest noise, every u = 1: every try starts at the
                # noise's last start (M - 1), which must not be clamped
                st.picks[0].copy_(longest)
                st.u[0].fill_(1.0)
            st.plan.run()
            snaps.append(st.snap())
        assert st.plan.is_graph()
        torch.cuda.synchronize()
        R.check_device_errors()
        total = near = 0
        outcomes = set()
        for r, snap in enumerate(snaps):
            c, n = check_snap(snap, spk, noi, Tm, LEN, -40.0, "run %d" % r)
            total, near = total + c, near + n
            used = snap["used"].cpu().numpy()
            outcomes |= {"first" if v == 1 else "later" if v > 1 else "none" for v in used}
        assert int(snaps[0]["starts"][0]) == noi[0].N - LEN
        assert near <= 0.05 * (total + near), (near, total)
        assert total >= 150
        assert {"first", "later"} <= outcomes, outcomes
    finally:
        st.plan.close()


def test_all_silent_takes_the_last_try(world, pools):
    """A threshold no crop reaches: used == 0 and the last try's start, with channel tables (D = C * len)."""
    render, R = _R()
    spk, noi = world
    _, sc, npool, _, Tc = pools
    st = Step(R, render, sc, npool, B=4, thr=100.0, tries=37, mono=False)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(12)
    try:
        for run in range(3):
            st.fill(gen, len(spk), len(noi))
            st.plan.run()
            snap = st.snap()
            torch.cuda.synchronize()
            assert (snap["used"] == 0).all()
            for b in range(4):
                p0, p1, pn = (int(v) for v in snap["picks"][b])
                M = min(spk[p0].N, spk[p1].N, noi[pn].N) - LEN + 1
                assert int(snap["starts"][b]) == dr.start_of(float(snap["u"][b, -1]), M)
            check_snap(snap, spk, noi, Tc, 2 * LEN, 100.0, "silent run %d" % run)
        R.check_device_errors()
    finally:
        st.plan.close()


def _bits(st):
    return [t.clone() for t in [st.starts, st.used, st.rms, st.mix] + st.outs]


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert torch.equal(x.nan_to_num(), y.nan_to_num())


def test_launches_no_graph_and_profiling(world, pools):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    spk, noi = world
    sm, _, npool, _, _ = pools
    st = Step(R, render, sm, npool, B=4)
    bare = R.plan_device(st.srcs, [torch.empty_like(o) for o in st.outs], mixtures=st.mixtures)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(13)
    try:
        st.fill(gen, len(spk), len(noi))
        st.plan.run()
        ref = _bits(st)
        c0 = R.launch_count()
        st.plan.run()
        with_draws = R.launch_count() - c0
        _same(ref, _bits(st))
        bare.run()
        c0 = R.launch_count()
        bare.run()
        assert with_draws == R.launch_count() - c0 + 1
        assert st.plan.is_graph() and bare.is_graph()
        # profiling: the same bits
        for o in st.outs + [st.rms, st.mix]:
            o.fill_(NAN)
        st.starts.fill_(-1)
        st.used.fill_(-1)
        R.set_profiling(True)
        try:
            st.plan.run()
            R.get_profile()
        finally:
            R.set_profiling(False)
        _same(ref, _bits(st))
    finally:
        st.plan.close()
        bare.close()
    # a context created under SS_NO_GRAPH, with its own banks and pools: the launches enqueued at every run, same bits
    ctx2 = ctypes.c_void_p()
    os.environ["SS_NO_GRAPH"] = "1"
    try:
        L.check(R.lib.ss_create(R.device, ctypes.byref(ctx2)))
    finally:
        del os.environ["SS_NO_GRAPH"]
    R2 = render.Renderer(R.device)
    R2.ctx = ctx2
    banks2 = []

    def moved(c):
        bank = R2.rir_bank(to(c.h))
        banks2.append(bank)
        return (render.MovingSource(to(c.x), bank, to(c.b), c.b) if c.b is not None
                else render.StaticSource(to(c.x), bank))
    sm2 = R2.source_pool([moved(c) for c in spk], levels="mono")
    np2 = R2.source_pool([moved(c) for c in noi])
    st2 = Step(R2, render, sm2, np2, B=4)
    try:
        st2.picks.copy_(st.picks)
        st2.u.copy_(st.u)
        st2.plan.run()
        assert not st2.plan.is_graph()
        _same(ref, _bits(st2))
    finally:
        st2.plan.close()
        sm2.close()
        np2.close()
        for b in banks2:
            b.close()
        R2.lib.ss_destroy(ctx2)


def test_side_stream_behind_queued_work(world, pools):
    render, R = _R()
    spk, noi = world
    sm, _, npool, Tm, _ = pools
    st = Step(R, render, sm, npool, B=8)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(14)
    try:
        st.plan.run()                                     # captured; the values below are new
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        assert s.cuda_stream != 0
        with torch.cuda.stream(s):
            for o in st.outs:
                o.fill_(NAN)
            st.u.fill_(0.5)
            st.picks.fill_(0)
            torch.cuda._sleep(SLEEP)
            st.picks[:, :2].copy_(torch.randint(0, len(spk), (8, 2), generator=gen, device="cuda", dtype=torch.int32))
            st.picks[:, 2].copy_(torch.randint(0, len(noi), (8,), generator=gen, device="cuda", dtype=torch.int32))
            st.u.uniform_(generator=gen)
            st.plan.run(stream=s.cuda_stream)
            busy = not s.query()
            snap = st.snap()
        assert busy
        s.synchronize()
        c, n = check_snap(snap, spk, noi, Tm, LEN, -40.0, "side stream")
        assert c + n == 8 and c >= 6
        R.check_device_errors()
    finally:
        st.plan.close()


def test_refusals(world, pools):
    from sonicsim_b200 import _lib as L
    render, R = _R()
    spk, noi = world
    sm, _, npool, _, _ = pools
    plain = R.source_pool([c.src for c in spk])
    st = Step(R, render, sm, npool, B=2, draws=False)
    start, u, used = st.starts[0], st.u[0], st.used[0]
    st.starts.fill_(-3)
    st.used.fill_(-7)
    S, O, M = st.srcs, st.outs, st.mixtures
    CD = render.CropDraw

    def py(draws, match, srcs=None, outs=None, mixtures=M):
        with pytest.raises(ValueError, match=match):
            R.plan_device(srcs or S, outs or O, mixtures=mixtures, draws=draws)

    try:
        py([CD(start, [0, 1], u[:0])], "u of draw 0")
        py([CD(start, [0, 1], torch.zeros(4097, dtype=torch.float64, device="cuda"))], "u of draw 0")
        py([CD(start, [0, 1], u.float())], "u of draw 0")
        py([CD(start, [], u)], "1 to 8 speakers")
        py([CD(start, list(range(9)), u)], "1 to 8 speakers")
        py([CD(start, [0, 0], u)], "more than once")
        py([CD(start, [0, 9], u)], "names source 9")
        py([CD(start, [0, 3], u)], "does not take its window start")
        py([CD(start, [0, 2], u)], "no level tables")
        py([CD(start, [0, 1], u, threshold_db=float("inf"))], "finite")
        py([CD(start, [0, 1], u, used=start)], "is its start")
        py([CD(start, [0, 1], u), CD(start, [0, 1], st.u[1])], "shares its start")
        py([CD(start.cpu(), [0, 1], u)], "start of draw 0")
        # a reader that is not a pooled slot; readers of different lengths; more than 16 readers
        fixed = spk[0].src._replace(window=(start, LEN))
        py([CD(start, [0, 1], u)], "not a pooled slot", srcs=S[:2] + [fixed] + S[3:])
        short = S[:2] + [render.Pooled(npool, st.picks[0, 2], (start, LEN - 1))] + S[3:]
        py([CD(start, [0, 1], u)], "different window lengths", srcs=short,
           outs=O[:2] + [torch.empty((2, LEN - 1), device="cuda")] + O[3:], mixtures=None)
        many = S + [render.Pooled(npool, st.picks[0, 2], (start, LEN)) for _ in range(14)]
        py([CD(start, [0, 1], u)], "at most 16", srcs=many, outs=O + [torch.empty_like(O[0]) for _ in range(14)])

        # the C ABI, past the Python checks
        items, n, keep = R._device_items(S, O)
        mixes = R._device_mixes(M, O, keep)
        good = R._device_draws([CD(start, [0, 1], u, used)], S, keep)

        def c_call(draws, nd=None, its=items, want=L.SS_ERR_INVALID):
            h = ctypes.c_void_p()
            got = R.lib.ss_plan_create_ex(R.ctx, its, n, mixes, len(mixes), draws, len(draws) if nd is None else nd,
                                          ctypes.byref(h))
            assert got == want and not h.value, (got, want)

        def variant(**kw):
            a = (L.SsPlanDraw * 1)()
            ctypes.memmove(a, good, ctypes.sizeof(L.SsPlanDraw))
            for k, v in kw.items():
                if k == "speakers":
                    for i, x in enumerate(v):
                        a[0].speakers[i] = x
                else:
                    setattr(a[0], k, v)
            return a

        h = ctypes.c_void_p()
        assert R.lib.ss_plan_create_ex(R.ctx, items, n, mixes, len(mixes), good, 1, ctypes.byref(h)) == 0
        R.lib.ss_plan_destroy(h)
        c_call(variant(S=9), want=L.SS_ERR_UNSUPPORTED)
        c_call(variant(tries=4097), want=L.SS_ERR_UNSUPPORTED)
        c_call((L.SsPlanDraw * 65536)(), want=L.SS_ERR_UNSUPPORTED)
        c_call(variant(S=0))
        c_call(variant(tries=0))
        c_call(variant(speakers=[0, 6]))
        c_call(variant(speakers=[-1, 1]))
        c_call(variant(speakers=[1, 1]))
        c_call(variant(speakers=[0, 2]))                  # a noise: a pool without levels
        c_call(variant(speakers=[0, 3]))                  # another example's start
        c_call(variant(start=None))
        c_call(variant(u=None))
        c_call(variant(threshold_db=float("nan")))
        c_call(variant(used=u.data_ptr()))                 # written over u
        c_call(variant(used=O[4].data_ptr()))              # over an output
        c_call(variant(used=st.rms.data_ptr()))            # over a mixture's rms_db
        c_call(variant(used=st.sirs.data_ptr()))           # over a mixture's sirs
        c_call(variant(used=st.picks.data_ptr()))          # over a pick
        c_call(variant(used=st.starts[1].data_ptr()))      # over another example's start
        two = (L.SsPlanDraw * 2)()
        ctypes.memmove(two, good, ctypes.sizeof(L.SsPlanDraw))
        ctypes.memmove(ctypes.byref(two, ctypes.sizeof(L.SsPlanDraw)), good, ctypes.sizeof(L.SsPlanDraw))
        two[1].used = None
        c_call(two)                                       # two draws, one start
        # a speaker of a pool without tables
        its = (L.SsSource * n)()
        ctypes.memmove(its, items, ctypes.sizeof(L.SsSource) * n)
        its[1].pool = plain._h.value
        c_call(good, its=its)
        # a reader that is not pooled: the noise slot as a fixed moving window at the draw's start
        its2 = (L.SsSource * n)()
        ctypes.memmove(its2, items, ctypes.sizeof(L.SsSource) * n)
        fx, _, _ = R._device_items([spk[0].src._replace(window=(start, LEN))], [O[2]])
        its2[2] = fx[0]
        c_call(good, its=its2)
        torch.cuda.synchronize()
        assert (st.starts == -3).all() and (st.used == -7).all()
    finally:
        plain.close()
