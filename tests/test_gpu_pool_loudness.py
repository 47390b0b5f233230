"""Loudness gains of source pools (Renderer.source_pool(..., lufs_targets=); ss_pool_loudness) through the real kernels.
SonicSet stores every stem loudness-normalised over the whole stem; a pool with gains makes every pooled slot render
the crop of that normalised stem.  Checked:
  1. SourcePool.loudness equals, bit for bit, the (LUFS, gain) render_host(..., lufs_targets=) measures for every
     candidate on its own, and the float64 BS.1770 oracle within 1e-6 dB; a silent candidate (-inf, measured as -40)
     and an unmeasured one (None: NaN, gain 1) included;
  2. every pooled output, direct stems included, equals the slice at its start of the candidate's whole normalised stem
     from render_host(..., lufs_targets=), bit for bit, over many runs with new picks and starts and NaN-filled outputs:
     an aligned speaker pool with direct stems, a static noise pool, a long-RIR pool, and a grid pool whose windows
     cover blocks that straddle waypoints (the fused red_add branch);
  3. the level tables of a gain pool are the float64 prefix sums of the normalised stems;
  4. a training plan over gain pools (pooled slots, mixtures, start draws) matches the draw and mix references on
     slices of the normalised stems, and a quiet candidate whose gain turns a silent crop into an accepted one keeps a
     different start than the same plan without gains;
  5. a plan over gain pools launches exactly what the same plan over the pools without gains launches, as a graph;
  6. every refusal, in Python and through the C ABI (each malformed field of a target's entry included), leaves the
     pool unchanged."""

import numpy as np
import pytest
import torch

from oracle import sonicsim_oracle as so
import draw_reference as dr
from draw_reference import Step, TABLE_TOL, TRIES, check_snap, gappy_dry
from gpu_plumbing import _R
from loudness_cases import MALFORMED
from pool_worlds import Cand, _mix_dev, fold_dev, gain_pool
from window_cases import _choice

pytestmark = pytest.mark.gpu

RATE = 16000
NAN = float("nan")
B = 4096


def speakers(seed, n=4, taps=40):
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        P, N = 3 + j % 3, 40000 + 5003 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        assert _choice(b, N, P, 4096) == 1
        x = so.synth_dry(rng, N) * np.float32(0.05 * (j + 1))
        if j == 1:
            x[:] = 0.0                                   # silent: -inf LUFS, measured as -40
        out.append(Cand(x, so.synth_rirs(rng, P, 2, 4096), b, taps))
    return out


def noises(seed, n=3):
    rng = np.random.default_rng(seed)
    return [Cand(so.synth_dry(rng, 30000 + 3001 * j) * np.float32(0.3), so.synth_rirs(rng, 1, 2, 4096)[0], None)
            for j in range(n)]


def longs(seed, n=3):
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        P, N = 3 + j % 2, 26000 + 5003 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 1, 9000), b))
    return out


def grids(seed, n=3):
    """Moving candidates with many short segments (grid blocking on their own): most blocks straddle a waypoint."""
    rng = np.random.default_rng(seed)
    out = []
    for j in range(n):
        P, N = 40, 24000 + 3000 * j
        np.random.seed(seed + j)
        idx, _ = so.setup_dynamic_interp(so.synth_path(rng, P), N)
        b = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)
        assert _choice(b, N, P, 4096) == 0
        out.append(Cand(so.synth_dry(rng, N), so.synth_rirs(rng, P, 2, 4096), b))
    return out


def straddling(b, N, start, wl):
    """Blocks of the 4096 grid that meet [start, start + wl) and more than one segment of trajectory b."""
    n = 0
    for s in range(start // B * B, start + wl, B):
        e = min(s + B, N) - 1
        n += int(np.searchsorted(b, s, side="right") != np.searchsorted(b, e, side="right"))
    return n


def test_loudness_equals_the_host_path_and_the_oracle():
    render, R = _R()
    cands = speakers(1, taps=0)
    targets = [-17.0, -16.0, None, -19.0]
    pool, norm = gain_pool(R, render, cands, targets)
    try:
        L = pool.loudness
        assert L.shape == (4, 2) and L.dtype == np.float64
        assert np.isnan(L[2]).all()
        for i, (c, t, nc) in enumerate(zip(cands, targets, norm)):
            if t is None:
                continue
            assert (L[i, 0], L[i, 1]) == tuple(nc.loud), (i, L[i], nc.loud)            # -inf == -inf
            ref = so.bs1770_integrated_loudness(c.full.cpu().numpy().T.astype(np.float64), RATE, 0.4,
                                                up_to_8_channels=True)
            if i == 1:
                assert np.isneginf(L[i, 0]) and np.isneginf(ref)
                assert L[i, 1] == pytest.approx(10.0 ** ((t + 40.0) / 20.0), rel=1e-15)
            else:
                assert abs(L[i, 0] - ref) < 1e-6, (i, L[i, 0], ref)
        assert pool.nbytes == 40 * 4 + 4 * 4
    finally:
        pool.close()


class Slots:
    """k pooled slots with device starts over one pool; NaN-filled outputs."""

    def __init__(self, render, R, pool, wl, k, taps=0):
        self.wl, self.taps = wl, taps
        self.picks = torch.zeros(k, dtype=torch.int32, device="cuda")
        self.starts = torch.zeros(k, dtype=torch.int32, device="cuda")
        self.srcs = [render.Pooled(pool, self.picks[j], (self.starts[j], wl), taps) for j in range(k)]
        C = pool.C
        self.outs = [torch.empty((C, wl), device="cuda") for _ in range(k)]
        self.douts = [torch.empty((C, wl), device="cuda") for _ in range(k)] if taps else None
        self.plan = R.plan_device(self.srcs, self.outs, direct_outs=self.douts)

    def run(self, pk, st):
        self.picks.copy_(torch.tensor(pk, dtype=torch.int32))
        self.starts.copy_(torch.tensor(st, dtype=torch.int32))
        for o in self.outs + (self.douts or []):
            o.fill_(NAN)
        self.plan.run()
        torch.cuda.synchronize()


@pytest.mark.parametrize("kind", ["speakers", "noise", "long", "grid"])
def test_pooled_outputs_are_slices_of_the_normalised_stems(kind):
    render, R = _R()
    make = {"speakers": speakers, "noise": noises, "long": longs, "grid": grids}[kind]
    taps = 40 if kind == "speakers" else 0
    cands = make(20 + len(kind)) if kind != "speakers" else make(21, taps=taps)
    rng = np.random.default_rng(5)
    targets = [float(rng.uniform(-31, -15)) for _ in cands]
    if kind == "speakers":
        targets[3] = None                                # unmeasured: gain 1, the raw stem
    pool, norm = gain_pool(R, render, cands, targets, taps)
    wl = 2 * B + 1000 if kind != "grid" else 3 * B + 500
    sl = Slots(render, R, pool, wl, k=6, taps=taps)
    straddled = 0
    try:
        for run in range(8):
            pk = [int(v) for v in rng.integers(0, len(cands), 6)]
            st = [int(rng.integers(0, cands[p].N - wl + 1)) for p in pk]
            sl.run(pk, st)
            for j, (p, s) in enumerate(zip(pk, st)):
                nc = norm[p]
                assert torch.equal(sl.outs[j], nc.full[:, s:s + wl]), (kind, run, j, p, s)
                if taps:
                    assert torch.equal(sl.douts[j], nc.full_d[:, s:s + wl]), (kind, run, j, p, s)
                if kind == "grid":
                    straddled += straddling(cands[p].b, cands[p].N, s, wl)
        assert sl.plan.is_graph()
        if kind == "grid":
            assert straddled > 0, straddled
            assert all(v != 1.0 for v in pool.loudness[:, 1])
    finally:
        sl.plan.close()
        pool.close()


@pytest.mark.parametrize("levels", ["mono", "channels"])
def test_level_tables_describe_the_normalised_stems(levels):
    render, R = _R()
    cands = noises(31)
    targets = [-24.0, -27.5, -22.25]
    pool, norm = gain_pool(R, render, cands, targets, levels=levels)
    try:
        assert pool.nbytes == 40 * 3 + 4 * 3 + 8 * sum(c.N + 1 for c in cands) + 8 * 3
        for i, nc in enumerate(norm):
            q = pool.level_table(i).cpu().numpy()
            ref = dr.level_table(nc.full.cpu().numpy(), levels == "mono", np.longdouble)
            assert q.shape == (nc.N + 1,) and q[0] == 0.0
            err = float(np.max(np.abs(q.astype(np.longdouble) - ref)))
            assert err <= TABLE_TOL * float(ref[-1]), (levels, i, err / float(ref[-1]))
            assert float(ref[-1]) != float(dr.level_table(cands[i].full.cpu().numpy(), levels == "mono")[-1])
    finally:
        pool.close()


@pytest.fixture(scope="module")
def world():
    """Gappy moving speakers at speech-like levels and static noises, SonicSet's targets for each."""
    rng = np.random.default_rng(108)
    spk, noi = [], []
    for j in range(5):
        P, N = 3 + j % 3, 200000 + 37003 * j
        b = np.round(np.linspace(0, N, P)).astype(np.int32)
        x = gappy_dry(rng, N) * np.float32(0.02 * (j + 1))
        spk.append(Cand(x, so.synth_rirs(rng, P, 2, 4096), b))
    for j in range(3):
        noi.append(Cand(so.synth_dry(rng, 150000 + 97001 * j), so.synth_rirs(rng, 1, 2, 4096)[0], None))
    t_spk = list(rng.uniform(-19, -15, len(spk)))
    t_noi = list(rng.uniform(-26, -22, len(noi)))
    return spk, noi, t_spk, t_noi


def test_training_plan_over_gain_pools(world):
    render, R = _R()
    spk, noi, t_spk, t_noi = world
    sm, nspk = gain_pool(R, render, spk, t_spk, levels="mono")
    npool, nnoi = gain_pool(R, render, noi, t_noi)
    Ts = [sm.level_table(i).cpu().numpy() for i in range(sm.n)]
    st = Step(R, render, sm, npool, B=12)
    LEN = st.outs[0].shape[1]
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    checked = 0
    try:
        for run in range(6):
            st.fill(gen, len(spk), len(noi))
            st.sirs.uniform_(-6, 6, generator=gen)
            st.snr.uniform_(10, 20, generator=gen)
            st.plan.run()
            snap = st.snap()
            c, _ = check_snap(snap, nspk, nnoi, Ts, LEN, st.thr, "gain run %d" % run)
            checked += c
            picks, starts = snap["picks"].cpu().numpy(), snap["starts"].cpu().numpy()
            for b in range(st.B):
                s = int(starts[b])
                crops = [n.full[:, s:s + LEN] for n in (nspk[picks[b, 0]], nspk[picks[b, 1]], nnoi[picks[b, 2]])]
                spk_f = torch.stack([fold_dev(crops[0]), fold_dev(crops[1])])
                mix, spk_out = _mix_dev(R, spk_f, fold_dev(crops[2])[None], st.sirs[b], st.snr[b])
                assert torch.equal(st.mix[b], mix), (run, b)
                for k in range(2):
                    v = spk_f[k].double()
                    ref = 10.0 * np.log10(max(1e-20, float((v * v).mean())))
                    assert abs(float(snap["rms"][b, k]) - ref) < 1e-4, (run, b, k)
        assert checked > 40 and st.plan.is_graph()
    finally:
        st.plan.close()
        sm.close()
        npool.close()


def test_gain_changes_a_silence_decision():
    """A quiet speaker (about -60 dBFS): every crop of the raw stem is below -40 dB, every crop of the stem normalised to
    -17 LUFS is above it.  With gains the first try is kept; without them every try fails and the last one is kept."""
    render, R = _R()
    rng = np.random.default_rng(77)
    N, P = 120000, 3
    b = np.round(np.linspace(0, N, P)).astype(np.int32)
    quiet = Cand(so.synth_dry(rng, N) * np.float32(1e-3), so.synth_rirs(rng, P, 2, 4096), b)
    noise = Cand(so.synth_dry(rng, N), so.synth_rirs(rng, 1, 2, 4096)[0], None)
    results = {}
    for gains in (True, False):
        sp = R.source_pool([quiet.src], levels="mono", lufs_targets=[-17.0] if gains else None)
        npool = R.source_pool([noise.src])
        st = Step(R, render, sp, npool, B=1)
        try:
            st.picks.zero_()
            st.u[0].copy_(torch.linspace(0.05, 0.95, TRIES, dtype=torch.float64))
            st.plan.run()
            torch.cuda.synchronize()
            results[gains] = (int(st.starts[0]), int(st.used[0]))
        finally:
            st.plan.close()
            sp.close()
            npool.close()
    M = N - 4 * RATE + 1
    assert results[True] == (dr.start_of(0.05, M), 1), results
    assert results[False] == (dr.start_of(0.95, M), 0), results


def test_launches_equal_the_plan_without_gains(world):
    render, R = _R()
    spk, noi, t_spk, t_noi = world
    counts = {}
    for gains in (True, False):
        sm = R.source_pool([c.src for c in spk], levels="mono", lufs_targets=t_spk if gains else None)
        npool = R.source_pool([c.src for c in noi], lufs_targets=t_noi if gains else None)
        st = Step(R, render, sm, npool, B=4)
        try:
            st.plan.run()
            torch.cuda.synchronize()
            R.reset_stats()
            st.plan.run()
            torch.cuda.synchronize()
            counts[gains] = (R.launch_count(), st.plan.is_graph())
        finally:
            st.plan.close()
            sm.close()
            npool.close()
    assert counts[True] == counts[False] and counts[True][1], counts


def _post(n, N, targets, rates):
    from sonicsim_b200 import _lib
    from sonicsim_b200.SonicSim_audio import gating_plan
    post = (_lib.SsPostLufs * n)()
    keep = []
    for i in range(n):
        if targets[i] is None:
            continue
        brk, blo, bhi = gating_plan(N[i], float(rates[i]), 0.4)
        keep.append((brk, blo, bhi))
        post[i] = _lib.SsPostLufs(brk=brk.ctypes.data, blk_lo=blo.ctypes.data, blk_hi=bhi.ctypes.data,
                                  n_e=len(brk) - 1, n_blocks=len(blo), rate=float(rates[i]), block_size=0.4,
                                  target_lufs=float(targets[i]))
    return post, keep


def test_refusals_leave_the_pool_unchanged():
    from sonicsim_b200 import _lib
    render, R = _R()
    lib = R.lib
    cands = noises(41)
    N = [c.N for c in cands]
    INV, UNS = _lib.SS_ERR_INVALID, _lib.SS_ERR_UNSUPPORTED

    def state(p):
        return lib.ss_pool_bytes(p._h), p.loudness.tobytes()

    # Python: the wrong number of targets, before any C call
    with pytest.raises(ValueError, match="entries in lufs_targets"):
        R.source_pool([c.src for c in cands], lufs_targets=[-20.0])
    # C ABI: NULL pool / post, mixed rates, loudness twice, after levels, after a plan
    assert lib.ss_pool_loudness(None, None) == INV
    pool = R.source_pool([c.src for c in cands])
    try:
        before = state(pool)
        assert lib.ss_pool_loudness(pool._h, None) == INV
        post, keep = _post(3, N, [-20.0, -21.0, -22.0], [16000, 16000, 22050])
        assert lib.ss_pool_loudness(pool._h, post) == INV and state(pool) == before
        post, keep = _post(3, N, [-20.0, None, -22.0], [16000] * 3)
        assert lib.ss_pool_loudness(pool._h, post) == _lib.SS_OK
        assert lib.ss_pool_bytes(pool._h) == 40 * 3 + 4 * 3
        after = lib.ss_pool_bytes(pool._h)
        assert lib.ss_pool_loudness(pool._h, post) == INV and lib.ss_pool_bytes(pool._h) == after
    finally:
        pool.close()
    pool = R.source_pool([c.src for c in cands], levels="channels")
    try:
        before = state(pool)
        post, keep = _post(3, N, [-20.0] * 3, [16000] * 3)
        assert lib.ss_pool_loudness(pool._h, post) == INV and state(pool) == before
    finally:
        pool.close()
    pool = R.source_pool([c.src for c in cands])
    picks = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.empty((2, 1000), device="cuda")
    plan = R.plan_device([render.Pooled(pool, picks[0], (0, 1000))], [out])
    try:
        before = state(pool)
        post, keep = _post(3, N, [-20.0] * 3, [16000] * 3)
        assert lib.ss_pool_loudness(pool._h, post) == INV and state(pool) == before
        plan.run()
        torch.cuda.synchronize()
        assert torch.equal(out, cands[0].full[:, :1000])
    finally:
        plan.close()
        pool.close()
    # C > 8: ValueError in Python, SS_ERR_UNSUPPORTED through the C ABI
    rng = np.random.default_rng(9)
    wide = [Cand(so.synth_dry(rng, 9000), so.synth_rirs(rng, 1, 9, 300)[0], None)]
    with pytest.raises(ValueError, match="at most 8 channels"):
        R.source_pool([wide[0].src], lufs_targets=[-20.0])
    pool = R.source_pool([wide[0].src])
    try:
        before = state(pool)
        post, keep = _post(1, [9000], [-20.0], [16000])
        assert lib.ss_pool_loudness(pool._h, post) == UNS and state(pool) == before
    finally:
        pool.close()


@pytest.mark.parametrize("bad", list(MALFORMED))
def test_pool_loudness_refuses_each_malformed_entry(bad):
    """The last of three entries (the second has no target) has one malformed field: SS_ERR_INVALID, the pool's bytes
    and loudness unchanged, and the same pool then takes well-formed targets."""
    from sonicsim_b200 import _lib
    render, R = _R()
    lib = R.lib
    cands = noises(41)
    N = [c.N for c in cands]
    field, value = MALFORMED[bad]
    pool = R.source_pool([c.src for c in cands])
    try:
        before = (lib.ss_pool_bytes(pool._h), pool.loudness.tobytes())
        post, keep = _post(3, N, [-20.0, None, -22.0], [RATE] * 3)
        setattr(post[2], field, value)
        assert lib.ss_pool_loudness(pool._h, post) == _lib.SS_ERR_INVALID
        assert (lib.ss_pool_bytes(pool._h), pool.loudness.tobytes()) == before
        post, keep = _post(3, N, [-20.0, None, -22.0], [RATE] * 3)
        assert lib.ss_pool_loudness(pool._h, post) == _lib.SS_OK
    finally:
        pool.close()
