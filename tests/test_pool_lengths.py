"""Pools whose candidates differ in L (RIR length) on the CPU, through the kernels' own helpers (exported by
tests/emu/ss_emu_pool_lengths.cu):
  - the head of k_blocks over a pool whose candidates differ in K sets the slot's K, nb, h_rows = P*C*K_i and the direct
    set's offset from the picked candidate, and fill_items follows it (kparts, pstride); a uniform pool's slot keeps K;
  - pool_table_cap with each candidate's own K is the largest table any candidate needs at any start;
  - a K = 1 candidate of a pool with longer RIRs renders through k_render<LONG> with kparts = 1: bit for bit the render
    of its bank with exact-zero partitions appended, and within float32 rounding - not bit for bit - of the render of its
    RIRs zero-padded to the pool's longest L: that bank's forward transforms pair each partition-0 row with a padded
    partition, whose half spectrum then holds the rounding residue of its partner rather than zeros (DESIGN section 3)."""
import ctypes

import numpy as np
import pytest

from emu import build_emu
from oracle import sonicsim_oracle as so
from window_cases import B, KSPEC, _choice, _k, _needs_numpy, _p, _random_bounds


@pytest.fixture(scope="module")
def emu():
    return build_emu.load("ss_emu_pool_lengths")


def test_pick_sets_the_picked_candidates_partitions(emu):
    N = np.array([9000, 30000, 20000, 41000], np.int32)
    P = np.array([3, 5, 2, 4], np.int32)
    out = np.zeros(12, np.int32)
    for K, uniform in [(np.array([1, 3, 2, 4], np.int32), 0), (np.array([2, 2, 2, 2], np.int32), 1)]:
        k_pool = int(K.max())
        for C in (1, 3):
            for direct in (0, 1):
                for v in (-1, 0, 1, 2, 3, 4):
                    for blk in (0, 1, 5):
                        emu.emu_pick_parts(v, 4, _p(N), _p(P), _p(K), uniform, k_pool, C, direct, blk, _p(out))
                        i = min(max(v, 0), 3)
                        Ki = int(K[i])
                        rows = int(P[i]) * C * Ki
                        want = [i, Ki, int(N[i]), int(P[i]), (int(N[i]) + B - 1) // B, rows, rows, min(Ki, blk + 1),
                                C * Ki, Ki if C > 1 else 0, rows if direct else 0, int(v != i)]
                        assert out.tolist() == want, (K.tolist(), C, direct, v, blk)


def test_table_cap_with_each_candidates_own_k(emu):
    """Random pools, L per candidate from {1000, 4096, 4097, 9000, 16384}: aligned only when every candidate would
    choose it with its own K; the table is the largest _needs_numpy of any candidate with its own K at any start."""
    rng = np.random.default_rng(21)
    lengths = [1000, 4096, 4097, 9000, 16384]
    seen = set()
    for case in range(30):
        static = case % 5 == 4
        cands = []
        for _ in range(int(rng.integers(2, 6))):
            L = int(rng.choice(lengths[:2] if case % 3 == 0 else lengths))
            P = 1 if static else int(rng.integers(2, 6 if case % 2 else 24))
            N = int(rng.integers(max(P, 6000), 50000))
            b = None if static else _random_bounds(rng, P, N, short=case % 2 == 0 and bool(rng.integers(0, 3) == 0))
            cands.append((N, P, b, L))
        aligned = 0 if static else int(all(_choice(b, N, P, L) for N, P, b, L in cands))
        Ks = np.array([_k(c[3]) for c in cands], np.int32)
        seen.add((aligned, len(set(Ks.tolist())) > 1))
        wl = int(rng.integers(1, min(c[0] for c in cands) + 1))
        need = max(int(_needs_numpy(N, b, aligned, _k(L), wl).max()) for N, P, b, L in cands)
        Na = np.array([c[0] for c in cands], np.int32)
        Pa = np.array([c[1] for c in cands], np.int32)
        if static:
            got = emu.emu_pool_table_cap_parts(None, None, _p(Na), _p(Pa), _p(Ks), len(cands), aligned, wl)
        else:
            off = np.cumsum([0] + [c[1] for c in cands[:-1]]).astype(np.int64)
            flat = np.ascontiguousarray(np.concatenate([c[2] for c in cands]), np.int32)
            got = emu.emu_pool_table_cap_parts(_p(flat), _p(off), _p(Na), _p(Pa), _p(Ks), len(cands), aligned, wl)
        assert got == need, (case, aligned, Ks.tolist(), wl)
        # the pool's K for every candidate sizes for more blocks in front: never less
        uni = max(int(_needs_numpy(N, b, aligned, int(Ks.max()), wl).max()) for N, P, b, L in cands)
        assert need <= uni
    assert (0, True) in seen and (1, False) in seen, seen


def _bank(emu, h):
    """The emulated bank (P*C*K, 4096) complex64 of RIRs h (P, C, L) (emu_bank_create of ss_emu_bank.cu)."""
    P, C, L = h.shape
    spec = np.full((P * C * _k(L), KSPEC), np.nan, np.complex64)
    emu.emu_bank_create(_p(h), P, C, L, 0, 0, _p(spec), None)
    assert not np.isnan(spec.view(np.float32)).any()
    return spec


def _render(emu, x, spec, bounds, P, C, L, mode, ws, wl, long_variant):
    out = np.full((C, wl), np.nan, np.float32)
    emu.emu_render_slot(_p(x), _p(spec), _p(out), _p(bounds), len(x), P, C, L, mode, ws, wl, long_variant)
    assert not np.isnan(out).any()
    return out


@pytest.mark.parametrize("mode, P, C, L, L_max", [(0, 1, 2, 1000, 9000), (0, 1, 3, 4096, 16384),
                                                   (1, 3, 2, 2500, 4097), (1, 4, 1, 4096, 16384)])
def test_one_partition_candidate_through_the_long_kernel(emu, mode, P, C, L, L_max):
    rng = np.random.default_rng(L + L_max + C)
    N = 30000
    x = so.synth_dry(rng, N)
    h = so.synth_rirs(rng, P, C, L).astype(np.float32)
    bounds = np.round(np.linspace(0, N, P)).astype(np.int32) if mode else None
    K = _k(L_max)
    hp = np.zeros((P, C, L_max), np.float32)
    hp[..., :L] = h
    spec1 = _bank(emu, h)                              # (P*C, 4096): one partition per row
    spec_p = _bank(emu, hp)                            # (P*C*K, 4096): the zero-padded RIRs' own bank
    spec_z = np.zeros((P * C * K, KSPEC), np.complex64)
    spec_z[::K] = spec1                                # the candidate's bank with K - 1 zero partitions appended
    for ws, wl in [(0, 5000), (N // 2 - 77, 7000), (N - 6000, 6000), (0, N)]:
        y1 = _render(emu, x, spec1, bounds, P, C, L, mode, ws, wl, 1)
        yz = _render(emu, x, spec_z, bounds, P, C, L_max, mode, ws, wl, 1)
        yp = _render(emu, x, spec_p, bounds, P, C, L_max, mode, ws, wl, 1)
        # kparts = 1 against kparts = min(K, reach) over exact-zero partitions: the same bits
        assert np.array_equal(y1, yz), (ws, wl)
        # the padded RIRs' own bank: its padded partitions are not exact zeros (below)
        scale = float(np.abs(yp).max())
        assert np.abs(y1 - yp).max() <= 1e-5 * scale, (ws, wl, float(np.abs(y1 - yp).max()), scale)
    # why: a zero row transformed together with a nonzero partner gets that partner's rounding residue, not zeros
    residue = np.abs(spec_p.reshape(P * C, K, KSPEC)[:, 1:]).max()
    assert 0 < residue < 1e-6 * np.abs(spec1).max(), residue
