"""Moving windows (ss_source.win_start_dev) on the CPU: the table a moving window is given holds the blocks of every
start (window_table_cap of ss_phases.cuh, exported by tests/emu/ss_emu_moving.cu, against the table window_blocks finds
for each start, swept over every start); k_blocks' clamp of a start read from device memory; and the refusals of the
pure-host hook and of the Python layer."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from window_cases import B, CASES, _needs_numpy, make_case
from sonicsim_b200 import _lib


@pytest.fixture(scope="module")
def emu_moving():
    return build_emu.load("ss_emu_moving")


def _lengths(N):
    return sorted({n for n in (1, 100, B - 1, B, B + 1, 3 * B + 5, 10000, N // 2, N - 1, N) if 1 <= n <= N})


@pytest.mark.parametrize("name", list(CASES))
def test_table_cap_holds_every_start(emu_moving, name):
    mode, P, C, L, N, taps = CASES[name]
    _, _, _, _, bounds, _ = make_case(name)
    bounds = np.ascontiguousarray(bounds, np.int32) if mode == 1 else None
    bp = bounds.ctypes.data if bounds is not None else None
    K, nb = (L + B - 1) // B, (N + B - 1) // B
    for aligned in ([1, 0] if mode == 1 and K == 1 else [0]):
        for wl in _lengths(N):
            need = np.zeros(N - wl + 1, np.int32)
            emu_moving.emu_window_tables(bp, N, P, L, aligned, wl, need.ctypes.data)
            assert np.array_equal(need, _needs_numpy(N, bounds, aligned, K, wl)), (name, aligned, wl)
            # the full plan on the host (grid blocking; aligned blocking with bounds_host): exactly the largest table
            cap = emu_moving.emu_window_table_cap(bp, N, P, L, aligned, 1, wl)
            assert cap == need.max(), (name, aligned, wl, cap, need.max())
            if aligned:
                # aligned blocking over device-side bounds: the device bound, never below what a start needs
                dcap = emu_moving.emu_window_table_cap(bp, N, P, L, aligned, 0, wl)
                assert need.max() <= dcap <= nb + P - 1, (name, wl, dcap)
            else:
                assert cap <= min(nb, (wl + B - 1) // B + K + 2), (name, wl, cap)


def test_table_cap_of_many_trajectories(emu_moving):
    """Random trajectories, lengths and both blockings: the host-planned cap is the largest table over every start."""
    rng = np.random.default_rng(5)
    for case in range(40):
        P = int(rng.integers(2, 30))
        N = int(rng.integers(max(P, 2), 60000))
        cuts = np.sort(rng.integers(0, (min(N, 3000) if case % 3 == 0 else N) + 1, P - 2))
        bounds = np.ascontiguousarray(np.concatenate([[0], cuts, [N]]), np.int32)
        L = int(rng.choice([300, 4096, 4097, 20000]))
        K = (L + B - 1) // B
        wl = int(rng.integers(1, N + 1))
        for aligned in ([1, 0] if K == 1 else [0]):
            need = _needs_numpy(N, bounds, aligned, K, wl)
            cap = emu_moving.emu_window_table_cap(bounds.ctypes.data, N, P, L, aligned, 1, wl)
            assert cap == need.max(), (case, aligned, wl)


def test_clamp_of_a_device_start(emu_moving):
    N, wl = 20000, 4096
    bad = ctypes.c_int32()
    for v, want, flagged in [(0, 0, 0), (1, 1, 0), (N - wl, N - wl, 0), (N - wl + 1, N - wl, 1), (-1, 0, 1),
                             (-(1 << 31), 0, 1), ((1 << 31) - 1, N - wl, 1), (12345, 12345, 0)]:
        got = emu_moving.emu_clamp_win_start(v, N, wl, ctypes.byref(bad))
        assert (got, bad.value) == (want, flagged), v
    assert emu_moving.emu_clamp_win_start(7, 10, 10, ctypes.byref(bad)) == 0 and bad.value == 1
    assert emu_moving.emu_clamp_win_start(0, 10, 10, ctypes.byref(bad)) == 0 and bad.value == 0


def test_debug_plan_refuses_a_device_start():
    """ss_debug_plan plans on the host, which cannot know a start held in device memory."""
    lib = _lib.load()
    b = np.array([0, 5000, 10000], np.int32)
    item = _lib.SsSource(x=1, rir=1, out=1, bounds=b.ctypes.data, N=10000, P=3, C=2, L=300,
                         mode=_lib.SS_MOVING_BOUNDS, bounds_host=b.ctypes.data, win_start=0, win_len=100)
    out = np.zeros((16, 4), np.int32)
    assert lib.ss_debug_plan(ctypes.byref(item), out.ctypes.data, 16, None) > 0
    item.win_start_dev = 4096
    assert lib.ss_debug_plan(ctypes.byref(item), out.ctypes.data, 16, None) == _lib.SS_ERR_INVALID


def test_python_refuses_tensor_starts_off_the_device_path():
    torch = pytest.importorskip("torch")
    from sonicsim_b200 import render
    src = render.MovingSource(np.zeros(100, np.float32), np.zeros((3, 1, 4), np.float32), np.array([0, 50, 100]))
    one = torch.tensor(3, dtype=torch.int32)
    # the host paths: any tensor start
    for start in (one, torch.tensor([3], dtype=torch.int32)):
        with pytest.raises(ValueError):
            render._window(src._replace(window=(start, 5)), 0, 100)
    # the device path: dtype, element count, device, length
    for start in (torch.tensor(3, dtype=torch.int64), torch.tensor(3.0), torch.zeros(2, dtype=torch.int32),
                  torch.zeros((1, 2), dtype=torch.int32), torch.zeros(0, dtype=torch.int32), one):
        with pytest.raises(ValueError):
            render._window_dev(src._replace(window=(start, 5)), 0, 100, 0)
    for n in (0, 101):
        with pytest.raises(ValueError):
            render._window_dev(src._replace(window=(one, n)), 0, 100, 0)
    # int starts keep their meaning on the device path
    assert render._window_dev(src._replace(window=(7, 5)), 0, 100, 0) == (7, 5, 5, None)
    assert render._window_dev(src, 0, 100, 0) == (0, 0, 100, None)
