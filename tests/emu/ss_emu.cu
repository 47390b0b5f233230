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

static void cta_spectra(const Source& S, int local, const Tables& T) {
    std::vector<float2> smem(kPadF);
    std::vector<Regs32> R(kThreads);
    Row ra, rb;
    const int nh = spectra_pairs_h(S);
    if (local < nh) { ra = make_row_h(S, 2 * local); rb = make_row_h(S, 2 * local + 1); }
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

// k_blocks: block table, 1 / n_s table, dense item numbering (one source here)
static void emu_blocks(const Source& S) {
    int nblk = 0;
    if (S.aligned) {
        for (int sg = 0; sg < S.P - 1; ++sg) {
            const int b0 = S.bounds[sg], n_s = S.bounds[sg + 1] - b0;
            for (int q = 0; q < seg_blocks(n_s); ++q) {
                Block bk; bk.start = b0 + kB * q; bk.len = n_s - kB * q < kB ? n_s - kB * q : kB; bk.p_lo = sg; bk.p_hi = sg + 1;
                S.blocks[nblk++] = bk;
            }
        }
    } else {
        nblk = S.nb;
        for (int bi = 0; bi < nblk; ++bi) {
            Block bk; bk.start = bi * kB; bk.len = S.N - bi * kB < kB ? S.N - bi * kB : kB; bk.p_lo = 0; bk.p_hi = 0;
            S.blocks[bi] = bk;
        }
    }
    for (int bi = nblk; bi < S.nblk_max; ++bi) { Block z; z.start = 0; z.len = 0; z.p_lo = 0; z.p_hi = 0; S.blocks[bi] = z; }
    if (S.mode == MODE_MOVING_BOUNDS)
        for (int sg = 0; sg < S.P - 1; ++sg) S.rstep[sg] = 1.0 / (double)(S.bounds[sg + 1] - S.bounds[sg]);
    S.counts[0] = nblk;
    S.counts[1] = 0;
}

// k_prepare's range CTAs: position range of every block in use + its work items
static void prepare_ranges(const Source& S, RItem* items) {
    for (int blk = 0; blk < S.counts[0]; ++blk) {
        Block bk = S.blocks[blk];
        if (S.mode == MODE_MOVING_BOUNDS && !S.aligned) {
            bk.p_lo = seg_of(S.bounds, S.P - 1, bk.start);
            bk.p_hi = seg_of(S.bounds, S.P - 1, bk.start + bk.len - 1) + 1;
        } else if (S.mode == MODE_MOVING_INDEXED) {
            int pmin = 0x7fffffff, pmax = -1;
            for (int n = bk.start; n < bk.start + bk.len; ++n) { int v = S.idx[n]; pmin = v < pmin ? v : pmin; pmax = v > pmax ? v : pmax; }
            bk.p_lo = pmin < 0 ? 0 : pmin;
            bk.p_hi = pmax + 1 > S.P - 1 ? S.P - 1 : pmax + 1;
        }
        for (int lane = 0; lane < 32; ++lane) fill_items(S, items, blk, bk, lane, 32);
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

extern "C" {

// Emulate k_spectra + k_render for one source.  mode: 0 static, 1 bounds, 2 (idx, w).
int emu_render(const float* x, const float* rir, float* out, const int32_t* bounds, const int32_t* idx,
               const float* w, int N, int P, int C, int L, int mode) {
    const Tables& T = tables();
    Source S;
    memset(&S, 0, sizeof(S));
    S.x = x; S.rir = rir; S.out = out; S.bounds = bounds; S.idx = idx; S.w = w;
    S.N = N; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = (N + kB - 1) / kB; S.mode = mode;
    S.aligned = (mode == MODE_MOVING_BOUNDS && S.K == 1) ? 1 : 0;
    S.nblk_max = S.aligned ? S.nb + P - 1 : S.nb;
    std::vector<float2> hs((size_t)P * C * S.K * kSpec), xs((size_t)S.nblk_max * kSpec);
    std::vector<RItem> items(max_render_items(S));
    std::vector<Block> blocks(S.nblk_max);
    std::vector<double> rstep(P);
    int counts[2] = {0, 0};
    S.hspec = hs.data(); S.xspec = xs.data(); S.blocks = blocks.data(); S.rstep = rstep.data(); S.counts = counts;
    emu_blocks(S);
    const int ns = spectra_pairs_h(S) + spectra_pairs_x(S);
    for (int i = 0; i < ns; ++i) cta_spectra(S, i, T);
    prepare_ranges(S, items.data());
    const int nr = counts[0] * items_per_block(S);
    const int grid = nr < 3 ? nr : 3;              // a few persistent CTAs, each looping over many items
    for (int cta = 0; cta < grid; ++cta) {
        if (S.aligned || (mode == MODE_STATIC && S.K == 1)) cta_render_fast(items.data(), nr, cta, grid, T);
        else cta_render(items.data(), nr, cta, grid, T, false, S.K > 1);
    }
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
