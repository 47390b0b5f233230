"""Trajectories of pooled slots (render.Trajectory, ss_trajectory) on the CPU, through the kernels' own helpers (exported
by tests/emu/ss_emu_traj.cu):
  - (0, P - 1, 0) with the candidate's own bounds renders the bits of the slot without a trajectory;
  - a forward sub-path (a, b) with bounds B renders the bits of the candidate with bounds that are B over [a, b] and
    empty elsewhere, under aligned and grid blocking, at every window edge;
  - a reverse path renders the bits of the forward path over the same spectra stored in reverse position order;
  - an invalid path or bounds table falls back to the candidate's own forward path and reports bit 8;
  - traj_table_cap holds the blocks of adversarial bounds (every segment boundary straddling a block) at every start;
  - every Python refusal is a ValueError raised before any C call."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from oracle import sonicsim_oracle as so
from window_cases import B, KSPEC, _k, _needs_numpy, _p, _random_bounds

vp, i32 = ctypes.c_void_p, ctypes.c_int


@pytest.fixture(scope="module")
def emu():
    lib = build_emu.load("ss_emu_traj")
    lib.emu_traj_table_cap.argtypes = [vp, vp, vp, i32, i32, i32]
    lib.emu_traj_render.argtypes = [vp] * 6 + [i32] * 7 + [vp]
    return lib


def _bank(emu, h):
    P, C, L = h.shape
    spec = np.full((P * C * _k(L), KSPEC), np.nan, np.complex64)
    emu.emu_bank_create(_p(h), P, C, L, 0, 0, _p(spec), None)
    return spec


def _render(emu, x, spec, bounds, P, C, L, aligned, ws, wl, path=None, tb=None):
    out = np.full((C, wl), np.nan, np.float32)
    info = np.zeros(4, np.int32)
    emu.emu_traj_render(_p(x), _p(spec), _p(out), _p(bounds), None if path is None else _p(path),
                        None if tb is None else _p(tb), len(x), P, C, L, aligned, ws, wl, _p(info))
    assert not np.isnan(out).any()
    return out, info


def _case(seed, P, C, L, N, aligned):
    rng = np.random.default_rng(seed)
    x = so.synth_dry(rng, N)
    h = so.synth_rirs(rng, P, C, L).astype(np.float32)
    # aligned blocking needs K == 1; segments of at least a block keep the candidate's own plan aligned
    bounds = np.round(np.linspace(0, N, P)).astype(np.int32)
    return rng, x, h, bounds


def _padded(tb, p_max):
    out = np.full(p_max, -7, np.int32)                  # entries past b - a must not be read
    out[:len(tb)] = tb
    return out


def _windows(N, rng):
    wl = int(rng.integers(3000, N // 2))
    return [(0, wl), (N - wl, wl), (int(rng.integers(0, N - wl)), wl), (B - 1, wl), (0, N)]


CASES = [(1, 5, 2, 3000, 60000, 1), (2, 6, 1, 4096, 50000, 1), (3, 5, 2, 9000, 60000, 0), (4, 9, 3, 2500, 70000, 0)]


@pytest.mark.parametrize("seed, P, C, L, N, aligned", CASES)
def test_whole_path_is_the_slot_without_a_trajectory(emu, seed, P, C, L, N, aligned):
    rng, x, h, bounds = _case(seed, P, C, L, N, aligned)
    spec = _bank(emu, h)
    path = np.array([0, P - 1, 0], np.int32)
    for ws, wl in _windows(N, rng):
        want, _ = _render(emu, x, spec, bounds, P, C, L, aligned, ws, wl)
        got, info = _render(emu, x, spec, bounds, P, C, L, aligned, ws, wl, path, _padded(bounds, P))
        assert info.tolist()[0] == 0 and info[2] == P and info[3] == 0
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (ws, wl)


def _sub_bounds(rng, a, b, N):
    """b - a + 1 ascending bounds from 0 to N, some segments empty, some shorter than a block"""
    cuts = np.sort(rng.integers(0, N + 1, b - a - 1))
    if b - a > 2:
        cuts[0] = cuts[1]                                # an empty segment
    return np.concatenate([[0], cuts, [N]]).astype(np.int32)


@pytest.mark.parametrize("seed, P, C, L, N, aligned", CASES)
def test_forward_subpath_is_the_candidate_with_empty_segments_elsewhere(emu, seed, P, C, L, N, aligned):
    rng, x, h, bounds = _case(seed, P, C, L, N, aligned)
    spec = _bank(emu, h)
    for a, b in [(0, 1), (1, P - 1), (P - 2, P - 1), (1, P - 2), (0, P - 1)]:
        tb = _sub_bounds(rng, a, b, N)
        full = np.concatenate([np.zeros(a, np.int32), tb, np.full(P - 1 - b, N, np.int32)]).astype(np.int32)
        for ws, wl in _windows(N, rng):
            want, _ = _render(emu, x, spec, full, P, C, L, aligned, ws, wl)
            got, info = _render(emu, x, spec, bounds, P, C, L, aligned, ws, wl, np.array([a, b, 0], np.int32),
                                _padded(tb, P))
            assert info[0] == 0 and info[2] == b - a + 1
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (a, b, ws, wl)


@pytest.mark.parametrize("seed, P, C, L, N, aligned", CASES)
def test_reverse_path_is_the_forward_path_over_reversed_positions(emu, seed, P, C, L, N, aligned):
    rng, x, h, bounds = _case(seed, P, C, L, N, aligned)
    spec = _bank(emu, h)
    # the same spectra with their positions stored in reverse order (a bank built from h[::-1] pairs its rows
    # differently in its forward transforms, so its bits differ)
    spec_r = np.ascontiguousarray(spec.reshape(P, -1, KSPEC)[::-1].reshape(spec.shape))
    for a, b in [(0, P - 1), (1, P - 2), (0, 1), (P - 3, P - 1)]:
        tb = _sub_bounds(rng, a, b, N)
        for ws, wl in _windows(N, rng):
            got, info = _render(emu, x, spec, bounds, P, C, L, aligned, ws, wl, np.array([a, b, 1], np.int32),
                                _padded(tb, P))
            assert info[0] == 0 and info[3] == 1
            # visited position j is bank position b - j, i.e. position P - 1 - b + j of the reversed bank
            want, _ = _render(emu, x, spec_r, bounds, P, C, L, aligned, ws, wl,
                              np.array([P - 1 - b, P - 1 - a, 0], np.int32), _padded(tb, P))
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (a, b, ws, wl)


def test_invalid_trajectories_fall_back_and_report(emu):
    P, C, L, N = 5, 2, 3000, 40000
    rng, x, h, bounds = _case(9, P, C, L, N, 1)
    spec = _bank(emu, h)
    want, _ = _render(emu, x, spec, bounds, P, C, L, 1, 1000, 9000)
    good = _padded(_sub_bounds(rng, 1, 3, N), P)
    bad_paths = [(2, 2, 0), (3, 1, 0), (-1, 2, 0), (0, P, 0), (0, 2, 2), (0, 2, -1)]
    for p in bad_paths:
        got, info = _render(emu, x, spec, bounds, P, C, L, 1, 1000, 9000, np.array(p, np.int32), good)
        assert info[0] == 256 and info[2] == P and info[3] == 0, p
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), p
    for tb in [[1, 100, N], [0, 100, N - 1], [0, 30000, 20000, N]]:   # not from 0, not to N, descending
        tb = np.array(tb, np.int32)
        path = np.array([0, len(tb) - 1, 1], np.int32)
        got, info = _render(emu, x, spec, bounds, P, C, L, 1, 1000, 9000, path, _padded(tb, P))
        assert info[0] == 256 and info[2] == P and info[3] == 0, tb
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), tb


def _straddling(rng, P_vis, N, wl):
    """Bounds of P_vis - 1 segments whose every inner boundary lies one sample past a block start of its segment's
    grid, so that each segment ends in a one-sample block: the most blocks a window of wl can meet."""
    seg = max(B + 1, wl // max(P_vis - 1, 1))
    cuts, at = [0], 0
    for _ in range(P_vis - 2):
        at = min(N, at + int(rng.choice([1, B + 1, 2 * B + 1, seg])))
        cuts.append(at)
    cuts.append(N)
    return np.array(cuts, np.int32)


def test_table_cap_holds_adversarial_bounds(emu):
    rng = np.random.default_rng(5)
    for case in range(40):
        n = int(rng.integers(1, 4))
        P = rng.integers(2, 40, n).astype(np.int32)
        N = rng.integers(20000, 200000, n).astype(np.int32)
        aligned = case % 4 != 3
        K = np.ones(n, np.int32) if aligned else rng.integers(1, 4, n).astype(np.int32)
        wl = int(rng.integers(1, int(N.min()) + 1)) if case % 5 else int(N.min())
        cap = emu.emu_traj_table_cap(_p(N), _p(P), _p(K), n, int(aligned), wl)
        for i in range(n):
            for trial in range(6):
                P_vis = int(rng.integers(2, P[i] + 1)) if trial else int(P[i])
                tb = _straddling(rng, P_vis, int(N[i]), wl) if trial % 2 == 0 else \
                    _random_bounds(rng, P_vis, int(N[i]), short=trial % 3 == 1) if P_vis > 2 else \
                    np.array([0, int(N[i])], np.int32)
                need = int(_needs_numpy(int(N[i]), tb, int(aligned), int(K[i]), wl).max())
                assert need <= cap, (case, i, P_vis, aligned, wl, need, cap)


def test_table_cap_is_the_pool_cap_under_grid_blocking(emu):
    rng = np.random.default_rng(6)
    for _ in range(20):
        n = int(rng.integers(1, 4))
        P = rng.integers(2, 30, n).astype(np.int32)
        N = rng.integers(10000, 90000, n).astype(np.int32)
        K = rng.integers(1, 4, n).astype(np.int32)
        wl = int(rng.integers(1, int(N.min()) + 1))
        want = max(int(_needs_numpy(int(N[i]), None, 0, int(K[i]), wl).max()) for i in range(n))
        assert emu.emu_traj_table_cap(_p(N), _p(P), _p(K), n, 0, wl) == want


def test_render_meets_the_table_cap(emu):
    """The window's table of an emulated run with adversarial drawn bounds fits traj_table_cap."""
    P, C, L, N = 7, 1, 3000, 90000
    rng, x, h, bounds = _case(11, P, C, L, N, 1)
    spec = _bank(emu, h)
    Na, Pa, Ka = np.array([N], np.int32), np.array([P], np.int32), np.ones(1, np.int32)
    for wl in (5000, 20000, N):
        cap = emu.emu_traj_table_cap(_p(Na), _p(Pa), _p(Ka), 1, 1, wl)
        tb = _straddling(rng, P, N, wl)
        for ws in (0, N - wl, (N - wl) // 2):
            _, info = _render(emu, x, spec, bounds, P, C, L, 1, ws, wl, np.array([0, P - 1, 0], np.int32), tb)
            assert info[0] == 0 and info[1] <= cap, (wl, ws, info.tolist(), cap)


# ---- refusals before any C call


class _Pool:
    """Stands for a SourcePool in refusals that never reach the library."""

    def __init__(self, mode=1, resident="device", gains=False, p_max=5):
        self.mode, self.resident, self.gains, self.p_max = mode, resident, gains, p_max


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError("a refusal reached the C ABI (%s)" % name)


def _renderer():
    from sonicsim_b200 import render
    R = object.__new__(render.Renderer)
    R.lib, R.device, R.ctx = _NoLib(), 0, None
    return R


def test_refusals_come_before_any_c_call():
    from sonicsim_b200 import render
    R = _renderer()
    t = render.Trajectory(None, None)
    win = (0, 1000)
    cases = [
        ([render.Pooled(_Pool(mode=0), None, win, trajectory=t)], None, "static pool"),
        ([render.Pooled(_Pool(resident="host"), None, win, trajectory=t)], None, "host pool"),
        ([render.Pooled(_Pool(gains=True), None, win, trajectory=t)], None, "loudness gains"),
        ([render.Pooled(_Pool(), None, win, dry=render.DryPick(None, None, gains=object()), trajectory=t)], None,
         "pair gains"),
        ([render.Pooled(_Pool(), None, win, trajectory=t)], [render.CropDraw(None, [0], None)], "CropDraw speaker"),
        ([render.Pooled(_Pool(), None, win, trajectory=(None, None))], None, "must be a Trajectory"),
        ([render.Pooled(_Pool(), None, win, trajectory=t)], None, "CUDA tensor"),
    ]
    for sources, draws, what in cases:
        with pytest.raises(ValueError, match=what):
            R._device_trajectories(sources, draws, ())


def test_no_trajectory_needs_nothing():
    from sonicsim_b200 import render
    R = _renderer()
    assert R._device_trajectories([render.Pooled(_Pool(), None, (0, 10))], None, ()) is None


def test_abi_layout():
    from sonicsim_b200 import _lib
    assert ctypes.sizeof(_lib.SsTrajectory) == 24
    assert [f[0] for f in _lib.SsTrajectory._fields_] == ["slot", "path_dev", "bounds_dev"]
    assert "ss_plan_create_traj" in _lib.EXPORTS
