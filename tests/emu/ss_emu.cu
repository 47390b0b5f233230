// tests/emu/ss_emu.cu - CPU emulation of the CUDA kernels, one emulated thread at a time.
//
// TEST INFRASTRUCTURE (not a product path, never shipped as a fallback).  It includes the very
// same per-thread phase functions the kernels call (sonicsim_b200/csrc/ss_phases.cuh) and replaces
// __syncthreads() by "finish the phase for every tid".  This is how index math, butterfly
// constants and the overlap-save / hat-weight logic are validated in the GPU-less authoring
// container.  Built with g++ (`-x c++`) into tests/emu/libss_emu.so by tests/emu/build.py.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"
#include "../../sonicsim_b200/csrc/ss_loud.cuh"

using namespace ss;

struct HostTables {
    std::vector<float2> tw, tb, tc;
    Tables T;
    HostTables() : tw(kF), tb(kTabB), tc(kTabC) {
        for (int m = 0; m < kF; ++m) {
            double a = -2.0 * M_PI * (double)m / (double)kF;
            tw[m] = make_float2((float)cos(a), (float)sin(a));
        }
        for (int r = 0; r < 16; ++r) {
            for (int k = 0; k < 16; ++k) {
                double a = -2.0 * M_PI * (double)(k * r) / 256.0;
                tb[r * 16 + k] = make_float2((float)cos(a), (float)sin(a));
            }
            for (int k = 0; k < 256; ++k) {
                double a = -2.0 * M_PI * (double)(k * r) / 4096.0;
                tc[r * 256 + k] = make_float2((float)cos(a), (float)sin(a));
            }
        }
        T.tw = tw.data(); T.twB = tb.data(); T.twC = tc.data();
    }
};
static const Tables& tables() { static HostTables h; return h.T; }

// k_rir_absmax (all partial maxima in slot 0) and k_rir_direct, one emulated lane per row; as in the kernels, a banked
// source (no rir) has its cuts already
static void emu_rir_prep(const Source& S, float* norm_part) {
    if (S.norm_part) {
        float m = 0.f;
        for (size_t i = 0; i < (size_t)S.P * S.C * S.L; ++i) m = fabsf(S.rir[i]) > m ? fabsf(S.rir[i]) : m;
        for (int i = 0; i < kNormParts; ++i) norm_part[i] = i == 0 ? m : 0.f;
    }
    if (S.cut && S.rir) {
        const float div = S.norm_part ? rir_absmax(S) : 0.f;
        for (int row = 0; row < S.P * S.C; ++row)
            S.cut[row] = direct_cut(peak_scan(S.rir + (size_t)row * S.L, S.L, div, 0, 1).i, S.L, S.direct_taps);
    }
}

// one k_prepare spectra CTA, rows chosen as the kernel chooses them (reverberant pairs, then direct pairs, then dry
// windows)
static void cta_spectra(const Source& S, int local, const Tables& T) {
    std::vector<float2> smem(kPadF);
    std::vector<Regs32> R(kThreads);
    Row ra, rb;
    const int nh = spectra_pairs_h(S);
    if (local < nh) rows_of_pair_h(S, local, ra, rb);
    else { local -= nh; ra = make_row_x(S, 2 * local); rb = make_row_x(S, 2 * local + 1); }
    if (!ra.dst && !rb.dst) return;
    float2* s = smem.data();
    for (int t = 0; t < kThreads; ++t) spectra_phase1(t, ra, rb, s);
    for (int t = 0; t < kThreads; ++t) load2(t, s, R[t]);
    for (int t = 0; t < kThreads; ++t) passB2<false>(t, s, R[t], T);
    for (int t = 0; t < kThreads; ++t) { load2(t, s, R[t]); spectra_phase3_compute(t, R[t], T); }
    for (int t = 0; t < kThreads; ++t) spectra_phase3_store(t, s, R[t]);
    for (int t = 0; t < kThreads; ++t) spectra_phase4(t, s, ra, rb);
}

// k_prepare's range warps: position range and work items of every block in use; a windowed source's blocks outside the
// window get no items
static void prepare_ranges(const Source& S, RItem* items) {
    for (int blk = 0; blk < S.counts[0]; ++blk) {
        if ((unsigned)(blk - win_first(S)) >= (unsigned)win_blocks(S)) continue;
        const Block bk = S.blocks[blk];
        int pmin = 0, pmax = 0;
        if (S.mode == MODE_MOVING_INDEXED) block_pos_scan(S, bk, 0, 1, pmin, pmax);
        fill_items(S, items, blk, block_positions(S, bk, pmin, pmax), 0, 1);
    }
}

// One persistent k_render CTA (`cta` of `grid`): same control flow as the kernel; the bulk copies
// are done at the point where thread 0 issues them, the mbarrier waits are no-ops.
static void cta_render(const RItem* items, int n_items, int cta, int grid, const Tables& T, bool fast, bool staged_long) {
    std::vector<float2> smem(kPadF + kSpec);
    std::vector<Regs32> R(kThreads);
    std::vector<DcNy> E(kThreads);
    float2* const fftbuf = smem.data();
    float2* const sX = fftbuf;
    float2* const sHp = fftbuf + kSpec;
    float2* const sHq = fftbuf + kPadF;
    RItem s_item[2];
    XDesc s_desc[2];
    int it_cur = cta, slot = 0, p_cur = 0;
    {
        XDesc d; memset(&d, 0, sizeof(d));
        if (it_cur < n_items) {
            s_item[0] = items[it_cur];
            if (it_cur + grid < n_items) s_item[1] = items[it_cur + grid];
            p_cur = s_item[0].p_lo;
            d = make_xdesc(s_item[0], p_cur);
        }
        s_desc[0] = d;
        if (d.valid) {
            memcpy(sX, d.X, sizeof(float2) * kSpec);
            memcpy(sHp, d.Hp, sizeof(float2) * kSpec);
            if (d.Hq) memcpy(sHq, d.Hq, sizeof(float2) * kSpec);
        }
    }
    for (int k = 0;; ++k) {
        const XDesc& d = s_desc[k & 1];
        if (!d.valid) break;
        if (fast) {
            for (int t = 0; t < kThreads; ++t) form_z<false, true>(t, sX, sHp, sHq, d, R[t]);          // k_render<false, true>
        } else if (d.kparts <= 1 && !staged_long) {
            for (int t = 0; t < kThreads; ++t) form_z<false, false>(t, sX, sHp, d.Hq ? sHq : nullptr, d, R[t]);
        } else if (!staged_long) {
            for (int t = 0; t < kThreads; ++t) form_z<true, false>(t, sX, sHp, d.Hq ? sHq : nullptr, d, R[t]);
        } else {                                                                                      // k_render<true, false>
            const float2* q = d.Hq ? sHq : nullptr;
            for (int t = 0; t < kThreads; ++t) long_stage<true>(t, sX, sHp, q, R[t], E[t]);
            for (int part = 1; part < d.kparts; ++part) {
                memcpy(sX, d.X - (size_t)part * kSpec, sizeof(float2) * kSpec);                      // thread 0's bulk copies
                memcpy(sHp, d.Hp + (size_t)part * kSpec, sizeof(float2) * kSpec);
                if (d.Hq) memcpy(sHq, d.Hq + (size_t)part * kSpec, sizeof(float2) * kSpec);
                for (int t = 0; t < kThreads; ++t) long_stage<false>(t, sX, sHp, q, R[t], E[t]);
            }
            for (int t = 0; t < kThreads; ++t) long_finish(t, R[t], E[t]);
        }
        {   // thread 0: publish transform k+1, stage its Hq
            XDesc nx; memset(&nx, 0, sizeof(nx));
            const RItem& cur = s_item[slot];
            if (p_cur + 2 <= cur.p_hi) { p_cur += 2; nx = make_xdesc(cur, p_cur); }
            else if (it_cur + grid < n_items) {
                it_cur += grid; slot ^= 1;
                p_cur = s_item[slot].p_lo;
                nx = make_xdesc(s_item[slot], p_cur);
                if (it_cur + grid < n_items) s_item[slot ^ 1] = items[it_cur + grid];
            }
            s_desc[(k + 1) & 1] = nx;
            if (nx.valid && nx.Hq) memcpy(sHq, nx.Hq, sizeof(float2) * kSpec);
        }
        for (int t = 0; t < kThreads; ++t) render_phase1(t, fftbuf, R[t]);
        for (int t = 0; t < kThreads; ++t) load2(t, fftbuf, R[t]);
        for (int t = 0; t < kThreads; ++t) passB2<true>(t, fftbuf, R[t], T);
        for (int t = 0; t < kThreads; ++t) load2(t, fftbuf, R[t]);
        const XDesc dcur = d;                      // (the device reads s_desc[k & 1] lazily; it is stable all iteration)
        {   // thread 0: stage X, Hp of transform k+1 into the (now free) FFT buffer
            const XDesc& nx = s_desc[(k + 1) & 1];
            if (nx.valid) { memcpy(sX, nx.X, sizeof(float2) * kSpec); memcpy(sHp, nx.Hp, sizeof(float2) * kSpec); }
        }
        for (int t = 0; t < kThreads; ++t) {
            render_phase3(t, R[t], T);
            if (fast) render_epilogue<true>(t, dcur, R[t]); else render_epilogue<false>(t, dcur, R[t]);
        }
    }
}

// One persistent k_render_fast CTA: the kernel's control flow with the split barriers collapsed (every phase runs for all
// threads before the next starts) and the bulk copies / item prefetches done at the points where the kernel issues them.
// As in the kernel: the CTA renders a contiguous range of items (per / rem), the filter spectra Hp, Hq land in the FFT
// buffer and the dry spectrum X in its own buffer behind it, X is copied only when the next item belongs to another
// block, and the inter-pass twiddles come from tw_get.
static void cta_render_fast(const RItem* items, int n_items, int cta, int grid, const Tables& T) {
    std::vector<float2> smem(kPadF + kSpec);
    std::vector<Regs32> R(kThreads);
    float2* const fftbuf = smem.data();
    float2* const sHp = fftbuf;
    float2* const sHq = fftbuf + kSpec;
    float2* const sX = fftbuf + kPadF;
    const int per = n_items / grid, rem = n_items % grid;
    const int n_k = per + (cta < rem ? 1 : 0);
    if (n_k <= 0) return;
    const RItem* my_items = items + (size_t)cta * per + (cta < rem ? cta : rem);
    RItem s_item[3];
    s_item[0] = my_items[0];
    if (n_k > 1) s_item[1] = my_items[1];
    {
        memcpy(sHp, item_hp(s_item[0]), sizeof(float2) * kSpec);
        memcpy(sHq, item_hq(s_item[0]), sizeof(float2) * kSpec);
        memcpy(sX, s_item[0].X, sizeof(float2) * kSpec);
    }
    XDesc unused; memset(&unused, 0, sizeof(unused)); unused.kparts = 1;
    std::vector<float2> w(kThreads * 16);
    for (int k = 0; k < n_k; ++k) {
        for (int t = 0; t < kThreads; ++t) form_z<false, true>(t, sX, sHp, sHq, unused, R[t]);
        for (int t = 0; t < kThreads; ++t) { fft16<true>(R[t].a); fft16<true>(R[t].b); }
        // B1 (kItemLane): the next item's X only if it belongs to another block; item k + 2 into the ring
        if (k + 1 < n_k) {
            const RItem& nx = s_item[(k + 1) % 3];
            if (nx.X != s_item[k % 3].X) memcpy(sX, nx.X, sizeof(float2) * kSpec);
        }
        if (k + 2 < n_k) s_item[(k + 2) % 3] = my_items[k + 2];
        for (int t = 0; t < kThreads; ++t) { passA_store(fftbuf, passA_jA(t), R[t].a); passA_store(fftbuf, passA_jB(t), R[t].b); }
        for (int t = 0; t < kThreads; ++t) load2(t, fftbuf, R[t]);
        for (int t = 0; t < kThreads; ++t) {
            float2 (&wt)[16] = *reinterpret_cast<float2 (*)[16]>(&w[16 * t]);
            tw_get<true, 16>(T.twB + (t & 15), wt);
            fft16_w<true>(R[t].a, wt); fft16_w<true>(R[t].b, wt);
        }
        for (int t = 0; t < kThreads; ++t) { passB_store(fftbuf, t, R[t].a); passB_store(fftbuf, t + 256, R[t].b); }
        for (int t = 0; t < kThreads; ++t) {
            load2(t, fftbuf, R[t]);
            float2 (&wt)[16] = *reinterpret_cast<float2 (*)[16]>(&w[16 * t]);
            tw_get<true, 256>(T.twC + t, wt);
        }
        if (k + 1 < n_k) {                          // last warp out of the FFT buffer: Hp, Hq of transform k + 1 into it
            const RItem& nx = s_item[(k + 1) % 3];
            memcpy(sHp, item_hp(nx), sizeof(float2) * kSpec);
            memcpy(sHq, item_hq(nx), sizeof(float2) * kSpec);
        }
        for (int t = 0; t < kThreads; ++t) {
            float2 (&wt)[16] = *reinterpret_cast<float2 (*)[16]>(&w[16 * t]);
            fft16_w<true>(R[t].a, wt); fft16_w<true>(R[t].b, wt);
            render_phase3_close(t, R[t], T);
            render_epilogue_item(t, s_item[k % 3], R[t]);
        }
    }
}

// The launches of one emulated source, as the library runs them: k_rir_absmax / k_rir_direct, the block table (k_blocks;
// windowed, win_len > 0: the full plan's blocks [g0, g1) that window_blocks finds), k_prepare's spectra CTAs and range
// warps, and the render CTAs.  aligned: the blocking plan.  rir == null: a banked source, spectra (and cuts) from
// bank / bank_cut.  direct_taps > 0: a direct-path stem into out_direct.  restrict_rows (windowed, with rir): transform
// only the RIR rows of the positions the window's blocks touch, else all of them.  win_stats (may be null) receives
// [table blocks, kept blocks, first RIR row, RIR rows per set], bank_stats (may be null) [RIR pair CTAs of k_prepare,
// dry-window pair CTAs, render items].
static void emu_source(const float* x, const float* rir, const float2* bank, const int* bank_cut, float* out,
                       const int32_t* bounds, const int32_t* idx, const float* w, int N, int P, int C, int L, int mode,
                       int aligned, int win_start, int win_len, float* out_direct, int direct_taps, int normalize,
                       int restrict_rows, int* win_stats, int* bank_stats) {
    const Tables& T = tables();
    Source S;
    memset(&S, 0, sizeof(S));
    S.x = x; S.rir = rir; S.out = out; S.bounds = bounds; S.idx = idx; S.w = w;
    S.N = N; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = (N + kB - 1) / kB; S.mode = mode;
    S.aligned = aligned;
    const bool windowed = win_len > 0;
    S.nblk_max = table_cap(aligned, S.nb, P);
    WinSpan ws = {0, S.nblk_max, 0, 0};
    if (windowed) {
        std::vector<Block> full(S.nblk_max);
        const int nfull = plan_blocks(aligned, bounds, P, N, S.nb, 0, S.nblk_max, full.data());
        ws = window_blocks(full.data(), nfull, win_start, win_start + win_len, S.K);
        S.nblk_max = ws.g1 - ws.g0;
    }
    std::vector<Block> blocks(S.nblk_max);
    const int nfull = plan_blocks(aligned, bounds, P, N, S.nb, ws.g0, ws.g1, blocks.data());
    const int nblk = (nfull < ws.g1 ? nfull : ws.g1) - ws.g0;
    clear_blocks(blocks.data(), nblk, S.nblk_max, 0, 1);
    std::vector<double> rstep(P);
    if (mode == MODE_MOVING_BOUNDS) fill_rstep(bounds, P, rstep.data(), 0, 1);
    int counts[8] = {nblk, 0, ws.k0 - ws.g0, ws.k1 - ws.k0, win_start, win_len, 0, 0};
    S.blocks = blocks.data(); S.rstep = rstep.data(); S.counts = counts;
    std::vector<float2> hs, xs((size_t)S.nblk_max * kSpec);
    std::vector<float> norm_part(kNormParts);
    std::vector<int> cut((size_t)P * C);
    if (rir) {
        if (normalize) S.norm_part = norm_part.data();
        if (direct_taps > 0) S.cut = cut.data();
        if (windowed) {                           // RIR positions the kept blocks interpolate between
            int pa = 0, pb = P - 1;
            if (mode == MODE_STATIC) pb = 0;
            else if (restrict_rows && mode == MODE_MOVING_BOUNDS) {
                pa = block_positions(S, blocks[counts[2]], 0, 0).p_lo;
                pb = block_positions(S, blocks[counts[2] + counts[3] - 1], 0, 0).p_hi;
            }
            window_rows(P, C, S.K, pa, pb, S.h_row0, S.h_rows);
        }
        hs.resize((size_t)(S.cut ? 2 : 1) * rows_stored_h(S) * kSpec);
        S.hspec = hs.data();
    } else {
        set_banked(S, const_cast<float2*>(bank), direct_taps > 0 ? const_cast<int*>(bank_cut) : nullptr, windowed);
    }
    if (direct_taps > 0) { S.out_direct = out_direct; S.direct_taps = direct_taps; }
    S.xspec = xs.data();
    std::vector<RItem> items(max_render_items(S));
    emu_rir_prep(S, norm_part.data());
    const int ns = spectra_pairs_h(S) + spectra_pairs_x(S);
    for (int i = 0; i < ns; ++i) cta_spectra(S, i, T);
    prepare_ranges(S, items.data());
    const int nr = win_blocks(S) * items_per_block(S);
    const int grid = nr < 3 ? nr : 3;              // a few persistent CTAs, each looping over many items
    for (int cta = 0; cta < grid; ++cta) {
        if (one_transform_per_item(S.aligned, mode, S.K)) cta_render_fast(items.data(), nr, cta, grid, T);
        else cta_render(items.data(), nr, cta, grid, T, false, S.K > 1);
    }
    if (win_stats) { win_stats[0] = S.nblk_max; win_stats[1] = ws.k1 - ws.k0; win_stats[2] = S.h_row0; win_stats[3] = S.h_rows; }
    if (bank_stats) { bank_stats[0] = spectra_pairs_h(S); bank_stats[1] = spectra_pairs_x(S); bank_stats[2] = nr; }
}

extern "C" {

// Emulate k_spectra + k_render for one source.  mode: 0 static, 1 bounds, 2 (idx, w).  Aligned blocking for every
// bounds trajectory with one RIR partition.
int emu_render(const float* x, const float* rir, float* out, const int32_t* bounds, const int32_t* idx,
               const float* w, int N, int P, int C, int L, int mode) {
    const int aligned = mode == MODE_MOVING_BOUNDS && (L + kB - 1) / kB == 1;
    emu_source(x, rir, nullptr, nullptr, out, bounds, idx, w, N, P, C, L, mode, aligned, 0, 0, nullptr, 0, 0, 0,
               nullptr, nullptr);
    return 0;
}

// forward 8192-point FFT of z = a + i b via the spectra kernel phases; returns the two half spectra
int emu_spectra_pair(const float* a, const float* b, int len, float* specA, float* specB) {
    const Tables& T = tables();
    Source S; memset(&S, 0, sizeof(S));
    std::vector<float> rir(2 * (size_t)len);
    memcpy(rir.data(), a, sizeof(float) * len); memcpy(rir.data() + len, b, sizeof(float) * len);
    S.rir = rir.data(); S.P = 1; S.C = 2; S.L = len; S.K = (len + kB - 1) / kB; S.N = 1; S.nb = 1; S.nblk_max = 0;
    std::vector<float2> hs((size_t)2 * S.K * kSpec);
    S.hspec = hs.data();
    for (int i = 0; i < spectra_pairs_h(S); ++i) cta_spectra(S, i, T);
    // return partition 0 of each row
    memcpy(specA, hs.data(), sizeof(float2) * kSpec);
    memcpy(specB, hs.data() + (size_t)S.K * kSpec, sizeof(float2) * kSpec);
    return 0;
}

// loudness: k_kweight_energy + k_loud_gate, one emulated thread per (channel, interval)
int emu_lufs(const float* data, int N, int C, long long stride_n, long long stride_c, double rate, double block_size,
             double target, const int32_t* brk, int n_e, const int32_t* blk_lo, const int32_t* blk_hi, int n_blocks,
             double* result) {
    LoudItem it; memset(&it, 0, sizeof(it));
    std::vector<double> E((size_t)kLoudScratch * C * n_e);
    it.data = data; it.brk = brk; it.blk_lo = blk_lo; it.blk_hi = blk_hi; it.E = E.data(); it.result = result;
    it.stride_n = stride_n; it.stride_c = stride_c; it.N = N; it.C = C; it.n_e = n_e; it.n_blocks = n_blocks;
    it.inv_norm = 1.0 / (block_size * rate); it.target = target;
    KCoef k = make_kcoef(rate);
    for (int c = 0; c < C; ++c) for (int e = 0; e < n_e; ++e) kweight_pass<1>(it, k, c, e);
    for (int c = 0; c < C; ++c) kw_scan_serial(it, c, 0);
    for (int c = 0; c < C; ++c) for (int e = 0; e < n_e; ++e) kweight_pass<2>(it, k, c, e);
    for (int c = 0; c < C; ++c) kw_scan_serial(it, c, 1);
    for (int c = 0; c < C; ++c) for (int e = 0; e < n_e; ++e) kweight_pass<3>(it, k, c, e);
    loudness_gate(it);
    return 0;
}

}  // extern "C"
