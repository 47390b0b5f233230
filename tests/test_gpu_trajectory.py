"""Trajectories of pooled slots (render.Trajectory) through the real kernels.  Checked:
  - (0, P - 1, 0) with the candidate's own bounds gives the bits of the same plan without trajectories: an aligned
    speaker pool with direct stems and a long-RIR grid pool, moving windows, dry picks;
  - a forward sub-path (a, b) with bounds B gives the bits of ss_render_dev of the candidate's bank with bounds that are
    B over [a, b] and empty elsewhere, direct stems included;
  - a reverse path matches the float64 render of the candidate's RIRs in reverse position order;
  - an invalid path or bounds table renders the candidate's own path and raises ValueError from check_device_errors;
  - launches per run are those of the plan without trajectories, and a side-stream run gives the same bits."""
import numpy as np
import pytest
import torch

from direct_path import direct_path_rirs
from gpu_plumbing import _R, to
from pool_worlds import TAPS, longs, speakers
from render_reference import TAU_GLOBAL, TAU_LOCAL, check_render, render_check_inputs
from window_cases import _choice

pytestmark = pytest.mark.gpu

NAN = float("nan")
WL = 9000


class Slots:
    """One pooled slot per candidate (pick j), moving starts, optional trajectories and dry picks."""

    def __init__(self, pool, cands, traj, taps=0, dry=None):
        render, R = _R()
        self.cands, self.taps = cands, taps
        n = len(cands)
        self.picks = torch.arange(n, dtype=torch.int32, device="cuda")
        self.starts = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.paths = torch.zeros((n, 3), dtype=torch.int32, device="cuda")
        self.bounds = torch.full((n, pool.p_max), -7, dtype=torch.int32, device="cuda")
        self.dpicks = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.srcs = []
        for j in range(n):
            t = render.Trajectory(self.paths[j], self.bounds[j]) if traj else None
            d = render.DryPick(dry, self.dpicks[j:j + 1]) if dry is not None else None
            self.srcs.append(render.Pooled(pool, self.picks[j:j + 1], (self.starts[j:j + 1], WL), taps, d, t))
        C = cands[0].C
        self.outs = [torch.full((C, WL), NAN, device="cuda") for _ in cands]
        self.douts = [torch.full((C, WL), NAN, device="cuda") for _ in cands] if taps else None
        self.plan = R.plan_device(self.srcs, self.outs, direct_outs=self.douts)

    def set(self, starts, paths=None, bounds=None, dpicks=None):
        self.starts.copy_(torch.tensor(starts, dtype=torch.int32))
        if paths is not None:
            self.paths.copy_(torch.tensor(np.array(paths), dtype=torch.int32))
            for j, b in enumerate(bounds):
                self.bounds[j, :len(b)] = torch.tensor(b, dtype=torch.int32)
        if dpicks is not None:
            self.dpicks.copy_(torch.tensor(dpicks, dtype=torch.int32))
        for o in self.outs + (self.douts or []):
            o.fill_(NAN)

    def run(self, stream=None):
        self.plan.run(stream)
        torch.cuda.synchronize()
        return [o.clone() for o in self.outs + (self.douts or [])]


def _starts(rng, cands):
    return [int(rng.choice([0, c.N - WL, rng.integers(0, c.N - WL + 1)])) for c in cands]


def _sub_bounds(rng, a, b, N):
    """b - a + 1 bounds from 0 to N in segments of similar length, one of them empty when there are three or more"""
    n = b - a
    w = rng.uniform(0.8, 1.2, n)
    if n > 2:
        w[1] = 0.0
    cum = np.concatenate([[0.0], np.cumsum(w)])
    return np.round(cum * (N / cum[-1])).astype(np.int32)


WORLDS = {"speakers": lambda: (speakers(31, n=4), TAPS), "long": lambda: (longs(32, n=3), 0)}


@pytest.mark.parametrize("kind", list(WORLDS))
def test_whole_path_is_the_plan_without_trajectories(kind):
    render, R = _R()
    cands, taps = WORLDS[kind]()
    pool = R.source_pool([c.src for c in cands])
    a, b = Slots(pool, cands, False, taps), Slots(pool, cands, True, taps)
    rng = np.random.default_rng(3)
    try:
        for run in range(4):
            st = _starts(rng, cands)
            a.set(st)
            b.set(st, [[0, c.h.shape[0] - 1, 0] for c in cands], [c.b for c in cands])
            for x, y in zip(a.run(), b.run()):
                assert torch.equal(x, y), (kind, run)
        R.check_device_errors()
        for p in (a, b):                      # launches per run are the plan's without trajectories
            p.plan.run()
            c0 = R.launch_count()
            p.plan.run()
            torch.cuda.synchronize()
            p.launches = R.launch_count() - c0
        assert a.launches == b.launches
        side = torch.cuda.Stream()            # a side-stream run gives the same bits
        ref = b.run()
        with torch.cuda.stream(side):
            for o in b.outs + (b.douts or []):
                o.fill_(NAN)
            b.plan.run(side.cuda_stream)
        side.synchronize()
        for x, y in zip(ref, b.outs + (b.douts or [])):
            assert torch.equal(x, y)
    finally:
        a.plan.close()
        b.plan.close()
        pool.close()


def test_whole_path_with_dry_picks():
    render, R = _R()
    cands = speakers(33, n=3, taps=0)
    pool = R.source_pool([c.src for c in cands])
    rng = np.random.default_rng(4)
    sig = [to(rng.standard_normal(max(c.N for c in cands) + 100).astype(np.float32) * 0.1) for _ in range(3)]
    dp = R.dry_pool(sig)
    a, b = Slots(pool, cands, False, dry=dp), Slots(pool, cands, True, dry=dp)
    try:
        for run in range(3):
            st, dk = _starts(rng, cands), rng.integers(0, 3, len(cands)).tolist()
            a.set(st, dpicks=dk)
            b.set(st, [[0, c.h.shape[0] - 1, 0] for c in cands], [c.b for c in cands], dk)
            for x, y in zip(a.run(), b.run()):
                assert torch.equal(x, y), run
    finally:
        a.plan.close()
        b.plan.close()
        dp.close()
        pool.close()


@pytest.mark.parametrize("kind", list(WORLDS))
def test_forward_subpath_is_the_candidate_with_empty_segments_elsewhere(kind):
    render, R = _R()
    cands, taps = WORLDS[kind]()
    pool = R.source_pool([c.src for c in cands])
    s = Slots(pool, cands, True, taps)
    rng = np.random.default_rng(5)
    try:
        for run in range(4):
            paths, tbs, fulls = [], [], []
            for c in cands:
                P = c.h.shape[0]
                a = int(rng.integers(0, P - 1))
                b = int(rng.integers(a + 1, P))
                tb = _sub_bounds(rng, a, b, c.N)
                full = np.concatenate([np.zeros(a, np.int32), tb, np.full(P - 1 - b, c.N, np.int32)]).astype(np.int32)
                paths.append([a, b, 0]); tbs.append(tb); fulls.append(full)
            st = _starts(rng, cands)
            s.set(st, paths, tbs)
            got = s.run()
            n = len(cands)
            refs = [torch.empty_like(o) for o in s.outs]
            drefs = [torch.empty_like(o) for o in s.outs] if taps else None
            R.render_device([c.src._replace(bounds=to(f), bounds_host=f, window=(w, WL), direct_taps=taps)
                             for c, f, w in zip(cands, fulls, st)], refs, direct_outs=drefs)
            torch.cuda.synchronize()
            for j, c in enumerate(cands):
                if kind == "speakers" and not _choice(fulls[j], c.N, c.h.shape[0], c.L):
                    # the candidate alone would take grid blocking over these bounds, the pool's slot stays aligned:
                    # the same samples within the float64 bounds instead of the same bits
                    y64, scale = render_check_inputs(c.x, c.h, 1, bounds=fulls[j], window=(st[j], WL))
                    check_render(got[j].cpu().numpy(), y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=st[j])
                    continue
                assert torch.equal(got[j], refs[j]), (kind, run, j, paths[j])
                if taps:
                    assert torch.equal(got[n + j], drefs[j]), (kind, run, j, "direct")
        R.check_device_errors()
    finally:
        s.plan.close()
        pool.close()


@pytest.mark.parametrize("kind", list(WORLDS))
def test_reverse_paths_against_float64(kind):
    render, R = _R()
    cands, taps = WORLDS[kind]()
    pool = R.source_pool([c.src for c in cands])
    s = Slots(pool, cands, True, taps)
    rng = np.random.default_rng(6)
    try:
        for run in range(3):
            paths, tbs = [], []
            for c in cands:
                P = c.h.shape[0]
                a = int(rng.integers(0, P - 1)) if run else 0
                b = int(rng.integers(a + 1, P)) if run else P - 1
                paths.append([a, b, 1]); tbs.append(_sub_bounds(rng, a, b, c.N))
            st = _starts(rng, cands)
            s.set(st, paths, tbs)
            got = s.run()
            for j, c in enumerate(cands):
                P = c.h.shape[0]
                a, b, _ = paths[j]
                # visited position k is position b - k: the forward path (P - 1 - b, P - 1 - a) over h[::-1]
                full = np.concatenate([np.zeros(P - 1 - b, np.int32), tbs[j],
                                       np.full(a, c.N, np.int32)]).astype(np.int32)
                y64, scale = render_check_inputs(c.x, np.ascontiguousarray(c.h[::-1]), 1, bounds=full,
                                                 window=(st[j], WL))
                check_render(got[j].cpu().numpy(), y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=st[j],
                             label="%s run %d slot %d path %s" % (kind, run, j, paths[j]))
                if taps:                      # the direct set follows the same map
                    h_d = direct_path_rirs(np.ascontiguousarray(c.h[::-1]), taps)
                    y64, scale = render_check_inputs(c.x, h_d, 1, bounds=full, window=(st[j], WL))
                    check_render(got[len(cands) + j].cpu().numpy(), y64, scale, TAU_LOCAL, TAU_GLOBAL, n0=st[j],
                                 label="%s run %d slot %d path %s direct" % (kind, run, j, paths[j]))
        R.check_device_errors()
    finally:
        s.plan.close()
        pool.close()


def test_invalid_trajectories_fall_back_and_raise():
    render, R = _R()
    cands = speakers(34, n=3, taps=0)
    pool = R.source_pool([c.src for c in cands])
    a, b = Slots(pool, cands, False), Slots(pool, cands, True)
    rng = np.random.default_rng(7)
    try:
        st = _starts(rng, cands)
        a.set(st)
        want = a.run()
        R.check_device_errors()
        bad = [([1, 1, 0], [0, 0]), ([0, 2, 2], [0, 10, 20]), ([0, 9, 0], [0, 10]), ([0, 1, 0], [5, 100])]
        for path, tb in bad:
            tb = [v if v != 20 else cands[0].N for v in tb]
            b.set(st, [path] + [[0, c.h.shape[0] - 1, 0] for c in cands[1:]], [tb] + [c.b for c in cands[1:]])
            got = b.run()
            for x, y in zip(want, got):
                assert torch.equal(x, y), path
            with pytest.raises(ValueError, match="Trajectory"):
                R.check_device_errors()
        b.set(st, [[0, c.h.shape[0] - 1, 0] for c in cands], [c.b for c in cands])
        b.run()
        R.check_device_errors()
    finally:
        a.plan.close()
        b.plan.close()
        pool.close()


def test_refusals_through_python():
    render, R = _R()
    cands = speakers(35, n=2, taps=0)
    pool = R.source_pool([c.src for c in cands])
    s = Slots(pool, cands, True)
    try:
        pick, start = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
        out = torch.empty((cands[0].C, WL), device="cuda")
        bad = [render.Trajectory(s.paths[0], s.bounds[0, :-1]),                  # not p_max entries
               render.Trajectory(s.paths[0].to(torch.int64), s.bounds[0]),        # not int32
               render.Trajectory(s.paths[0], out.view(-1)[:pool.p_max].view(torch.int32))]   # meets the output
        for t in bad:
            with pytest.raises(ValueError):
                R.plan_device([render.Pooled(pool, pick, (start, WL), trajectory=t)], [out])
        # one tensor object as a path and as a value draw's out: refused in Python, before any C call
        path = torch.zeros(3, dtype=torch.int32, device="cuda")
        rng = torch.zeros(2, dtype=torch.int64, device="cuda")
        c0 = R.launch_count()
        with pytest.raises(ValueError, match="trajectory of source 0 meets"):
            R.plan_device([render.Pooled(pool, pick, (start, WL), trajectory=render.Trajectory(path, s.bounds[1]))],
                          [out], values=[render.ValueDraw(path.view(1, 3), rng, 0, 2)])
        with pytest.raises(ValueError, match="trajectory of source 0 meets"):
            R.plan_device([render.Pooled(pool, pick, (start, WL), trajectory=render.Trajectory(path, s.bounds[1]))],
                          [out], values=[render.ValueDraw(path, rng, 0, 2)])
        assert R.launch_count() == c0
    finally:
        s.plan.close()
        pool.close()


RATE, N_EQ, M = 16000, 48000, 12


def _utterances(rng, n):
    """n 16-bit utterances of 0.2 to 1.3 s"""
    out = []
    for _ in range(n):
        v = rng.standard_normal(int(rng.integers(RATE // 5, int(1.3 * RATE)))) * rng.uniform(0.05, 0.5)
        out.append(np.clip(np.round(v * 32768), -32768, 32767).astype(np.int16))
    return out


def _layout(rng, lengths):
    ids, offs = np.full(M, -1, np.int32), np.full(M, -1, np.int32)
    pos = int(rng.integers(0, RATE))
    for e in range(M):
        if pos >= N_EQ:
            break
        i = int(rng.integers(0, len(lengths)))
        ids[e], offs[e] = i, pos
        pos += lengths[i] + int(rng.integers(0, RATE))
    return ids, offs


def _assemble(ids, offs, utts):
    x = np.zeros(N_EQ, np.float32)
    for i, o in zip(ids, offs):
        if i >= 0 and o < N_EQ:
            n = min(utts[i].size, N_EQ - o)
            x[o:o + n] = utts[i][:n].astype(np.float32) * np.float32(1 / 32768)
    return x


def test_loudness_stream_slots_measure_the_trajectorys_whole_stem():
    """Stream slots with StemLoudness and a forward sub-path on a grid-blocked pool (K = 3): every crop and (LUFS, gain)
    equals render_host(..., lufs_targets=) of the candidate with the dry stream and bounds that are the drawn ones over
    [a, b] and empty elsewhere, bit for bit - the whole stem is rendered and measured with the run's trajectory."""
    from pool_worlds import Cand
    from oracle import sonicsim_oracle as so
    render, R = _R()
    rng = np.random.default_rng(41)
    cands = [Cand(so.synth_dry(rng, N_EQ), so.synth_rirs(rng, P, 1, 9000),
                  np.round(np.linspace(0, N_EQ, P)).astype(np.int32)) for P in (3, 4, 5)]
    pool = R.source_pool([c.src for c in cands])
    utts = _utterances(rng, 6)
    upool = R.dry_pool(utts, dtype="int16")
    k, wl = 3, 16000
    d = "cuda"
    picks = torch.zeros(k, dtype=torch.int32, device=d)
    starts = torch.zeros(k, dtype=torch.int32, device=d)
    lay = torch.full((k, 2, M), -1, dtype=torch.int32, device=d)
    target = torch.zeros((k, 1), dtype=torch.float64, device=d)
    res = torch.full((k, 2), NAN, dtype=torch.float64, device=d)
    paths = torch.zeros((k, 3), dtype=torch.int32, device=d)
    tbounds = torch.zeros((k, pool.p_max), dtype=torch.int32, device=d)
    outs = [torch.empty((1, wl), device=d) for _ in range(k)]
    srcs = [render.Pooled(pool, picks[j:j + 1], (starts[j:j + 1], wl),
                          dry=render.DryStream(upool, lay[j, 0], lay[j, 1],
                                               lufs=render.StemLoudness(target[j], res[j], RATE)),
                          trajectory=render.Trajectory(paths[j], tbounds[j])) for j in range(k)]
    plan = R.plan_device(srcs, outs)
    try:
        for run in range(3):
            pk = rng.integers(0, len(cands), k)
            rows = [_layout(rng, [u.size for u in utts]) for _ in range(k)]
            st = rng.integers(0, N_EQ - wl + 1, k)
            tg = rng.uniform(-31.0, -15.0, k)
            fulls = []
            for j in range(k):
                c = cands[pk[j]]
                P = c.h.shape[0]
                a = int(rng.integers(0, P - 1))
                b = int(rng.integers(a + 1, P))
                tb = _sub_bounds(rng, a, b, N_EQ)
                paths[j] = torch.tensor([a, b, 0], dtype=torch.int32)
                tbounds[j, :len(tb)] = torch.from_numpy(tb)
                fulls.append(np.concatenate([np.zeros(a, np.int32), tb,
                                             np.full(P - 1 - b, N_EQ, np.int32)]).astype(np.int32))
                lay[j, 0] = torch.from_numpy(rows[j][0]); lay[j, 1] = torch.from_numpy(rows[j][1])
            picks.copy_(torch.from_numpy(pk.astype(np.int32)))
            starts.copy_(torch.from_numpy(st.astype(np.int32)))
            target.copy_(torch.from_numpy(tg[:, None]))
            for o in outs:
                o.fill_(NAN)
            plan.run()
            torch.cuda.synchronize()
            for j in range(k):
                c = cands[pk[j]]
                x = _assemble(rows[j][0], rows[j][1], utts)
                lo = []
                y = R.render_host([render.MovingSource(x, c.bank, fulls[j])], lufs_targets=[float(tg[j])],
                                  loudness_out=lo, sr=RATE)[0]
                s0 = int(st[j])
                assert torch.equal(outs[j].cpu(), torch.from_numpy(y[:, s0:s0 + wl])), (run, j)
                assert tuple(res[j].cpu().numpy()) == tuple(lo[0]), (run, j)
        R.check_device_errors()
    finally:
        plan.close()
        upool.close()
        pool.close()


def test_dry_picked_crop_draw_speakers_with_trajectories():
    """Dry-picked CropDraw speakers with the whole-path trajectory: starts, `used` and every crop equal the same plan
    without trajectories (a dry-picked speaker's level table is its dry signal's, which no trajectory changes)."""
    render, R = _R()
    cands = speakers(36, n=3, taps=0)
    pool = R.source_pool([c.src for c in cands])
    rng = np.random.default_rng(8)
    n_max = max(c.N for c in cands)
    sig = []
    for _ in range(3):
        v = rng.standard_normal(n_max + 50).astype(np.float32) * 0.1
        v[:int(rng.integers(1000, 20000))] = 0.0            # a silent head, so that some tries are rejected
        sig.append(to(v))
    dp = R.dry_pool(sig, levels=True)
    d = "cuda"
    runs = {}
    try:
        for traj in (False, True):
            picks = torch.tensor([0, 1, 2], dtype=torch.int32, device=d)
            dpicks = torch.zeros(3, dtype=torch.int32, device=d)
            start = torch.zeros(1, dtype=torch.int32, device=d)
            used = torch.zeros(1, dtype=torch.int32, device=d)
            u = torch.zeros(101, dtype=torch.float64, device=d)
            paths = torch.tensor([[0, c.h.shape[0] - 1, 0] for c in cands], dtype=torch.int32, device=d)
            tb = torch.full((3, pool.p_max), -7, dtype=torch.int32, device=d)
            for j, c in enumerate(cands):
                tb[j, :len(c.b)] = torch.from_numpy(c.b)
            srcs = [render.Pooled(pool, picks[j:j + 1], (start, WL), dry=render.DryPick(dp, dpicks[j:j + 1]),
                                  trajectory=render.Trajectory(paths[j], tb[j]) if traj else None) for j in range(3)]
            outs = [torch.full((cands[0].C, WL), NAN, device=d) for _ in range(3)]
            plan = R.plan_device(srcs, outs, draws=[render.CropDraw(start, [0, 1], u, used)])
            g = np.random.default_rng(9)
            snaps = []
            try:
                for run in range(4):
                    dpicks.copy_(torch.from_numpy(g.integers(0, 3, 3).astype(np.int32)))
                    u.copy_(torch.from_numpy(g.random(101)))
                    for o in outs:
                        o.fill_(NAN)
                    plan.run()
                    torch.cuda.synchronize()
                    snaps.append((int(start.item()), int(used.item()), [o.cpu().clone() for o in outs]))
                R.check_device_errors()
            finally:
                plan.close()
            runs[traj] = snaps
        for (s0, u0, o0), (s1, u1, o1) in zip(runs[False], runs[True]):
            assert (s0, u0) == (s1, u1)
            for x, y in zip(o0, o1):
                assert torch.equal(x, y)
    finally:
        dp.close()
        pool.close()
