"""16-bit dry pools (ss_dry_pool_create_i16; Renderer.dry_pool(..., dtype="int16")) on the CPU.
  - The exactness argument itself, in NumPy: the float32 square of k / 32768 is a multiple of 2^-30 and at most 1, so
    the float64 prefix sums of a signal of N <= 2^23 samples are the same in sequential, reversed and pairwise order -
    random int16 signals, and the worst case (every sample -32768, N = 2^23).
  - The sparse-table lookup of ss_phases.cuh (sparse_level, exported by tests/emu/ss_emu_compact.cu) and the host-side
    rebuild of DryPool.level_table (_levels_from_sparse) equal the full table at every start residue mod 64, at s = 0
    and at s = N.
  - k_draw<true>'s draws (draw_silent_i16 over the sparse table and the int16 samples) equal the float-table draws
    start for start and `used` for `used`, on streams built as create_long_audio builds them (utterances in zeros):
    crops that fall in the gaps, thresholds hit exactly, crops ending at N, float and 16-bit speakers in one draw; and
    the picked signal and table behind a 16-bit pool's pointer array (speaker_signal_i16), picks clamped.
  - k_stage<true>'s head and its int16 -> float32 staging give the float pool's staged samples and view, bit for bit,
    reading only whole groups of 4 inside the signal's 64-byte padded arena span.
  - The float -> int16 acceptance check of Renderer.dry_pool and its refusals, before any C call."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from sonicsim_b200 import render

B = 4096


def squares(k):
    """The float32 squares of k / 32768 as float64: the terms k_levels adds."""
    v = k.astype(np.float32) * np.float32(1.0 / 32768.0)
    return (v * v).astype(np.float64)


def full_table(k):
    """Q[0] = 0, Q[n + 1] = Q[n] + (double)(x[n] * x[n]), summed in order."""
    return np.concatenate([[0.0], np.cumsum(squares(k))])


def sparse_table(Q):
    N = Q.size - 1
    return Q[np.minimum(np.arange(-(-N // 64) + 1) * 64, N)].copy()


def pairwise_prefix(t):
    """Inclusive prefix sums by a Hillis-Steele tree: every sum in another grouping than the sequential one."""
    s = t.copy()
    o = 1
    while o < s.size:
        s[o:] = s[o:] + s[:-o].copy()
        o <<= 1
    return np.concatenate([[0.0], s])


def reversed_prefix(t):
    """Q[s] = total - (suffix sum from s), the suffix sums accumulated from the end."""
    suf = np.concatenate([np.cumsum(t[::-1])[::-1], [0.0]])
    return suf[0] - suf


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_compact")


def long_audio(rng, N, n_utt, amp=(0.01, 0.9)):
    """A stream as create_long_audio builds one: whole utterances (int16 noise of random level) placed into zeros,
    never overlapping, with exact-zero gaps between them."""
    k = np.zeros(N, np.int16)
    pos = 0
    for _ in range(n_utt):
        gap, length = int(rng.integers(0, N // (2 * n_utt))), int(rng.integers(64, N // (2 * n_utt)))
        a, b = pos + gap, min(N, pos + gap + length)
        if a >= N:
            break
        k[a:b] = np.clip(rng.standard_normal(b - a) * 32768 * rng.uniform(*amp), -32768, 32767).astype(np.int16)
        pos = b
    return k


# ------------------------------------------------------------------------------------------- the exactness argument
def test_squares_are_multiples_of_2_pow_minus_30():
    k = np.arange(-32768, 32768, dtype=np.int32).astype(np.int16)
    t = squares(k)
    assert t.max() == 1.0 and t.min() == 0.0
    assert np.all(t * 2.0 ** 30 == np.floor(t * 2.0 ** 30))


def test_prefix_sums_do_not_depend_on_the_order():
    rng = np.random.default_rng(1)
    for N in (1, 63, 64, 65, 4097, 1 << 20):
        k = rng.integers(-32768, 32768, N).astype(np.int16)
        t = squares(k)
        Q = full_table(k)
        assert np.array_equal(Q, pairwise_prefix(t))
        assert np.array_equal(Q, reversed_prefix(t))


def test_worst_case_signal_of_2_pow_23_samples():
    N = 1 << 23
    k = np.full(N, -32768, np.int16)
    t = squares(k)
    assert np.all(t == 1.0)
    Q = full_table(k)
    assert np.array_equal(Q, np.arange(N + 1, dtype=np.float64))
    assert np.array_equal(Q, reversed_prefix(t))
    assert np.array_equal(Q, pairwise_prefix(t))


# ------------------------------------------------------------------------------------------------ the sparse lookup
@pytest.mark.parametrize("N", [1, 5, 63, 64, 65, 127, 128, 4096 * 3 + 17])
def test_sparse_lookup_equals_the_full_table(emu, N):
    rng = np.random.default_rng(N)
    k = rng.integers(-32768, 32768, N).astype(np.int16)
    Q = full_table(k)
    q = sparse_table(Q)
    s = np.unique(np.concatenate([[0, N], np.arange(0, N + 1, max(1, N // 300)),
                                  [min(N, 64 * (N // 128) + r) for r in range(64)]])).astype(np.int32)
    out = np.empty(s.size)
    emu.emu_sparse_levels(q.ctypes.data, k.ctypes.data, s.ctypes.data, s.size, out.ctypes.data)
    assert np.array_equal(out, Q[s])
    assert set(np.asarray(s) % 64) >= set(range(min(64, N + 1)))       # every residue the signal has
    assert np.array_equal(render._levels_from_sparse(q, k), Q)


def test_host_rebuild_of_long_audio_tables():
    rng = np.random.default_rng(7)
    for N in (48000, 64 * 1000, 160000 + 3):
        k = long_audio(rng, N, 6)
        Q = full_table(k)
        assert np.array_equal(render._levels_from_sparse(sparse_table(Q), k), Q)


# ------------------------------------------------------------------------------------------------------ the draws
def _draw(emu, speakers, M, length, u, thr):
    """speakers: [(Q, q, k)] with k None for a float speaker (full table Q, D = len)."""
    S = len(speakers)
    Qp = (ctypes.c_void_p * S)(*[sp[0].ctypes.data for sp in speakers])
    qp = (ctypes.c_void_p * S)(*[sp[1].ctypes.data for sp in speakers])
    xp = (ctypes.c_void_p * S)(*[None if sp[2] is None else sp[2].ctypes.data for sp in speakers])
    D = np.full(S, float(length))
    used = ctypes.c_int32()
    u = np.ascontiguousarray(u, np.float64)
    s = emu.emu_draw_i16(ctypes.cast(Qp, ctypes.c_void_p), ctypes.cast(qp, ctypes.c_void_p),
                         ctypes.cast(xp, ctypes.c_void_p), D.ctypes.data, S, M, length, u.ctypes.data, u.size,
                         float(thr), ctypes.byref(used))
    return s, used.value


def _both(emu, sigs, M, length, u, thr, mixed=False):
    """The draw over float tables and over 16-bit speakers (every other one when mixed)."""
    tabs = [(full_table(k), k) for k in sigs]
    fl = [(Q, Q, None) for Q, _ in tabs]
    i16 = [(Q, sparse_table(Q), None if mixed and j % 2 else k) for j, (Q, k) in enumerate(tabs)]
    return _draw(emu, fl, M, length, u, thr), _draw(emu, i16, M, length, u, thr)


def test_draws_over_long_audio_equal_the_float_draws(emu):
    rng = np.random.default_rng(3)
    n_gap = 0
    for trial in range(40):
        N = int(rng.integers(20000, 90000))
        length = int(rng.choice([64, 1000, 4000, 16000]))
        sigs = [long_audio(rng, N, int(rng.integers(1, 6))) for _ in range(int(rng.integers(1, 4)))]
        M = N - length + 1
        u = rng.random(int(rng.integers(1, 200)))
        u[-1] = 1.0                                     # the last try ends at N
        for thr in (-200.0, -60.0, -35.0, -20.0, 0.0):
            a, b = _both(emu, sigs, M, length, u, thr)
            assert a == b, (trial, thr)
            a, b = _both(emu, sigs, M, length, u, thr, mixed=True)
            assert a == b, (trial, thr)
            if a[1] != 1:
                n_gap += 1
    assert n_gap > 20                                   # many draws rejected crops (gaps, quiet utterances)


def test_draw_thresholds_hit_exactly(emu):
    N, length = 4096, 256
    k = np.zeros(N, np.int16)
    k[2048:] = -32768                                   # v = -1: ms = 1, 0 dB exactly; zeros: ms = 1e-20, -200 dB
    M = N - length + 1
    u_gap, u_loud, u_end = 0.0, 2048.5 / M, 1.0
    for u, thr, silent in [(u_gap, -200.0, False), (u_gap, -199.0, True), (u_loud, 0.0, False), (u_loud, 1e-3, True),
                           (u_end, 0.0, False), (u_end, 1e-3, True)]:
        a, b = _both(emu, [k], M, length, [u], thr)
        assert a == b
        assert a[1] == (0 if silent else 1), (u, thr)


def test_picked_signal_and_table_behind_the_pointer_array(emu):
    n = 5
    xs = [np.full(10 + i, i, np.int16) for i in range(n)]
    qs = [np.full(3, float(i)) for i in range(n)]
    xp = (ctypes.c_void_p * n)(*[x.ctypes.data for x in xs])
    qp = (ctypes.c_void_p * n)(*[q.ctypes.data for q in qs])
    for v, want in [(0, 0), (3, 3), (4, 4), (5, 4), (1 << 30, 4), (-1, 0), (-(1 << 31), 0)]:
        out = np.zeros(2, np.int32)
        emu.emu_speaker_i16(ctypes.cast(xp, ctypes.c_void_p), ctypes.cast(qp, ctypes.c_void_p), n, v, out.ctypes.data)
        assert list(out) == [want, want], v


# ------------------------------------------------------------------------------------------------------ the staging
@pytest.mark.parametrize("P,K", [(1, 1), (1, 3), (5, 1), (9, 2)])
def test_staged_samples_equal_the_float_pool(emu, P, K):
    rng = np.random.default_rng(P * 10 + K)
    for trial in range(12):
        N = int(rng.integers(3 * B, 12 * B)) + int(rng.integers(0, 4))
        Nd = N + int(rng.integers(0, 70))
        k = long_audio(rng, Nd, 4)
        d = k.astype(np.float32) * np.float32(1.0 / 32768.0)
        bounds = np.sort(rng.choice(np.arange(1, N - 1), P - 2, replace=False)).astype(np.int32) if P > 2 else None
        bounds = np.concatenate([[0], [] if bounds is None else bounds, [N]]).astype(np.int32) if P > 1 else \
            np.zeros(1, np.int32)
        wl = int(rng.integers(1, N))
        for ws in {0, N - wl, int(rng.integers(0, N - wl + 1)), min(N - wl, (K + 2) * B)}:
            for dv in (0, 2, 7, -3):
                cap = Nd + 16
                of, oi = np.full(cap, np.nan, np.float32), np.full(cap, np.nan, np.float32)
                info = np.zeros(8, np.int32)
                emu.emu_stage_i16(bounds.ctypes.data, N, P, 2, K, ws, wl, d.ctypes.data, k.ctypes.data, Nd, 3, dv,
                                  of.ctypes.data, oi.ctypes.data, info.ctypes.data)
                x0, x1 = info[0], info[1]
                assert (info[2], info[3]) == (x0, x1) and x0 % 4 == 0 and x1 % 4 == 0 and x1 <= -(-N // 4) * 4
                assert info[4] == info[5] == (16 if dv in (7, -3) else 0)
                assert info[6] == 1 and info[7] == 1
                assert np.array_equal(of[:x1 - x0].view(np.uint32), oi[:x1 - x0].view(np.uint32))
                ref = np.zeros(x1 - x0, np.float32)
                ref[:max(0, min(Nd, x1) - x0)] = d[x0:min(Nd, x1)]
                assert np.array_equal(oi[:x1 - x0], ref)


# ------------------------------------------------------------------------------------------ acceptance and refusals
def test_accepted_inputs_convert_to_the_same_int16():
    rng = np.random.default_rng(5)
    k = rng.integers(-32768, 32768, 1000).astype(np.int16)
    k[:2] = (-32768, 32767)
    for x in (k, k.astype(np.float32) / np.float32(32768), k.astype(np.float64) / 32768.0, k[::1]):
        keep = []
        ptr, N = render._as_i16(x, "signal 0", 0, keep)
        assert N == k.size and keep[-1].dtype == np.int16 and np.array_equal(keep[-1], k)
        assert ptr == keep[-1].ctypes.data
    keep = []
    render._as_i16(k[::2], "signal 0", 0, keep)                # strided: copied contiguous
    assert keep[-1].flags.c_contiguous and np.array_equal(keep[-1], k[::2])


@pytest.mark.parametrize("x,match", [
    (np.array([0.0, 0.5, 1.0 / 65536], np.float64), "signal 3 has sample 2"),
    (np.array([0.0, 1.0], np.float32), "signal 3 has sample 1"),
    (np.array([-1.0 - 1.0 / 32768], np.float64), "signal 3 has sample 0"),
    (np.array([0.0, np.nan], np.float32), "signal 3 has sample 1"),
    (np.array([np.inf], np.float32), "signal 3 has sample 0"),
    (np.array([1, 2], np.int32), "int16 or float"),
    (np.array([1, 2], np.uint8), "int16 or float"),
    (np.array([True]), "int16 or float"),
    (np.zeros(0, np.int16), "1 to 2\\^23"),
    (np.zeros((2, 3), np.int16), "1-D"),
    (np.zeros((1 << 23) + 1, np.int16), "1 to 2\\^23"),
])
def test_refused_inputs(x, match):
    with pytest.raises(ValueError, match=match):
        render._as_i16(x, "signal 3", 0, [])


def test_longest_signal_is_accepted():
    keep = []
    _, N = render._as_i16(np.zeros(1 << 23, np.int16), "signal 0", 0, keep)
    assert N == 1 << 23
