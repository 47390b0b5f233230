// sonicsim_b200 :: ss_kernels.cu  -  sm_90a kernels + the C ABI of include/sonicsim_b200.h
//
// Path (SURVEY section 8a):  SonicSim_moving.convolve_moving_receiver (SonicSim_moving.py:63-96) and
// convolve_fixed_receiver (:47-61), restructured as a uniformly partitioned overlap-save
// convolution in the segment-local form
//      y[c,n] = sum_p hat_p(n) (x * h[p,c])[n],     hat_p = linear hat over segments p-1, p,
// so only the two positions a sample needs are ever convolved (2/P of the reference's work) and the
// (P, C, N) intermediate of :86 is never materialised.
//
// Launches per chunk of sources (DESIGN.md section 2):
//   k_blocks  : block table (waypoint-aligned or 4096-grid) + dense numbering of the work items; skipped
//               when the trajectory bounds are on the host, which then builds the same tables itself
//   k_prepare : real rows (RIR partitions, dry windows) -> half spectra (two rows per complex FFT);
//               one warp per block fills that block's k_render work items
//   k_render  : persistent CTAs; per transform Z = sum_part X[b-part] (H[p] + i H[p+1]) from spectra the
//               bulk-copy engine staged in shared memory one transform ahead; one 8192-point inverse FFT
//               gives both positions' convolutions as Re / Im; the closing radix-2 is fused with the
//               per-sample lerp and the (C, N) store.  <LONG>: RIR partitions >= 1 (staged one after the other).
//   k_render_fast : the same for all-aligned chunks (one item = one transform), see its own header below
//   k_rir_absmax  : optional, SS_RIR_NORMALIZE: global abs-max of a source's RIR tensor for k_prepare's row loads
//   k_rir_direct  : optional, SS_DIRECT_TARGET: per-row direct-path length (argmax |h| + direct_taps); k_prepare then
//                   transforms the truncated rows as a second RIR set and fills a second group of items per block
// A source with an RIR spectrum bank (ss_bank) has its RIR spectra (and cuts) already: it adds no k_rir_absmax /
// k_rir_direct work and no RIR CTAs to k_prepare.  A bank is built by these same launches over a source without blocks.
// Consecutive chunks rotate through three streams / scratch buffers so that they overlap; a bound batch (ss_plan_*)
// captures all of it into one CUDA graph.
// fp32 throughout (the reference is float32 end to end, SURVEY 8), no cuFFT.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <new>
#include <vector>

#include "ss_internal.h"
#include "ss_phases.cuh"
#include "ss_loud.cuh"

using namespace ss;

// Device-path trajectory check: the kernels cannot raise, so a source whose device-side trajectory breaks the contract
// of ss_render_dev (idx outside [0, P - 2]; bounds not ascending from 0 to N) sets a bit here; ss_device_errors reads
// and clears it.  bit 0: index out of range, bit 1: bounds not monotone / not ending at N, bit 2: a moving window's
// start outside [0, N - win_len] (clamped), bit 3: a pooled slot's pick outside [0, n) (clamped), bit 4: a dry pick
// outside [0, n) of its dry pool (clamped), bit 8: an invalid trajectory of a pooled slot (its candidate's own path used).
__device__ unsigned g_dev_err;

// twiddle tables, filled from the host in double precision (ss_create)
__device__ float2 g_tw[kF];          // exp(-2 pi i m / 8192)
__device__ float2 g_twB[kTabB];      // [r][k] exp(-2 pi i k r / 256)
__device__ float2 g_twC[kTabC];      // [r][k] exp(-2 pi i k r / 4096)

// ----------------------------------------------------------------------------- k_blocks
// One warp walks the aligned segments of S, 32 at a time: body(sg, b0, n_s, first) for every segment [b0, b0 + n_s)
// that has blocks, `first` = full-plan index of its first block (inclusive shuffle sum of seg_blocks).  Returns the
// full plan's block count.
template <class Body>
__device__ int seg_scan(const Source& S, int lane, Body body) {
    int carry = 0;
    for (int base = 0; base < S.P - 1; base += 32) {
        const int sg = base + lane;
        const int b0 = sg < S.P - 1 ? S.bounds[sg] : 0;
        const int n_s = sg < S.P - 1 ? S.bounds[sg + 1] - b0 : 0;
        const int cnt = n_s > 0 ? seg_blocks(n_s) : 0;
        int incl = cnt;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        if (cnt > 0) body(sg, b0, n_s, carry + incl - cnt);
        carry += __shfl_sync(0xffffffffu, incl, 31);
    }
    return carry;
}

// Windowed source: the full-plan blocks holding the window's first and last samples, then window_span.  The table never
// holds the full plan.
__device__ WinSpan window_blocks_dev(const Source& S, int lane) {
    const int ws = S.counts[4], we = ws + S.counts[5];
    if (!S.aligned) return window_span(ws / kB, (we + kB - 1) / kB, S.nb, S.K);
    int f0 = -1, f1 = -1;
    const int nfull = seg_scan(S, lane, [&](int sg, int b0, int n_s, int first) {
        if (ws >= b0 && ws < b0 + n_s) f0 = first + (ws - b0) / kB;
        if (we - 1 >= b0 && we - 1 < b0 + n_s) f1 = first + (we - 1 - b0) / kB;
    });
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        f0 = max(f0, __shfl_xor_sync(0xffffffffu, f0, o));
        f1 = max(f1, __shfl_xor_sync(0xffffffffu, f1, o));
    }
    const int k0 = f0 < 0 ? 0 : f0;               // (-1: a bounds table outside the contract; keep the writes in range)
    return window_span(k0, f1 < k0 ? k0 + 1 : f1 + 1, nfull, S.K);
}

// The full plan's blocks [g0, g1) into the table (one warp), the rest of the table cleared, 1 / n_s table, counts[0].
__device__ void write_blocks(const Source& S, int lane, int g0, int g1) {
    int nfull = S.nb;
    if (S.aligned) {
        nfull = seg_scan(S, lane, [&](int sg, int b0, int n_s, int first) {
            for (int q = 0; q < seg_blocks(n_s); ++q)
                if (first + q >= g0 && first + q < g1) S.blocks[first + q - g0] = seg_block(b0, n_s, q, sg);
        });
    } else {
        for (int bi = g0 + lane; bi < g1 && bi < S.nb; bi += 32) S.blocks[bi - g0] = grid_block(S.N, bi);
    }
    const int nblk = (g1 < nfull ? g1 : nfull) - g0;
    clear_blocks(S.blocks, nblk, S.nblk_max, lane, 32);
    if (S.mode == MODE_MOVING_BOUNDS) fill_rstep(S.bounds, S.P, S.rstep, lane, 32);
    if (lane == 0) S.counts[0] = nblk;
}

// One small CTA per chunk: block table of every source (one warp per source), 1 / n_s table, then the
// exclusive scan that packs the render work items of all sources into one dense table.  A whole source's table is the
// full plan; a windowed one's holds the full plan's blocks [g0, g1) (window_span, cut to the table size).  A moving
// window first reads its start from device memory, clamps it (bit 2 of g_dev_err) and stores it as counts[4], where
// the window search here and k_prepare's range warps take it; its table is sized for every start (window_table_cap).
// A pooled slot reads its pick before that, clamps it (bit 3) and writes the picked candidate - its RIR partition count
// when the pool's candidates differ in K (pick_parts), and its loudness gain, counts[11] - into its Source in the
// descriptor block (pick_slot), which is why k_prepare then reads the Source table from global memory (k_prepare<false>).
// A dry-picked slot then reads its dry pick, clamps it (bit 4) and puts the picked dry signal in place of x (pick_dry);
// with pair gains (ss_pair_gains) it takes the pair's gain in place of the candidate's.  A slot with a trajectory
// (ss_trajectory) then takes the run's path and bounds over the picked candidate (take_trajectory, bit 8), and after the
// scan its work items are filled here (fill_traj_items) instead of by k_prepare's range warps.
__global__ void __launch_bounds__(256)
k_blocks(Source* srcs, int n_src, int* __restrict__ total_items, RItem* __restrict__ items) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (int si = warp; si < n_src; si += nwarps) {
        Source& S = srcs[si];
        int g0 = 0, g1 = S.nblk_max;
        if (S.h_rows) {
            if (pool_table(S) && lane == 0) {
                const StageView* const sv = stage_view(S);
                if (sv) {
                    take_view(S, *sv);                  // a host pool: k_stage picked (bit 3) and staged the candidate
                } else {
                    const unsigned err = pick_pooled(S);   // the pick (bit 3), and a dry pick (bit 4)
                    if (err) atomicOr(&g_dev_err, err);
                }
                if (has_traj(S)) {                      // the run's trajectory over the picked candidate (bit 8)
                    const unsigned err = take_trajectory(S);
                    if (err) atomicOr(&g_dev_err, err);
                }
            }
            __syncwarp();
            const int* const ws_dev = win_start_ptr(S);
            if (ws_dev && lane == 0) {
                bool bad;
                S.counts[4] = clamp_win_start(*ws_dev, S.N, S.counts[5], bad);
                if (bad) atomicOr(&g_dev_err, 4u);
            }
            __syncwarp();
            const WinSpan w = window_blocks_dev(S, lane);
            g0 = w.g0;
            g1 = w.g1 - w.g0 > S.nblk_max ? w.g0 + S.nblk_max : w.g1;
            if (lane == 0) {
                S.counts[2] = w.k0 - w.g0;
                S.counts[3] = (w.k1 < g1 ? w.k1 : g1) - w.k0;
            }
        }
        write_blocks(S, lane, g0, g1);
    }
    __syncthreads();
    if (warp == 0) {
        int carry = 0;
        for (int base = 0; base < n_src; base += 32) {
            const int si = base + lane;
            const int cnt = si < n_src ? win_blocks(srcs[si]) * items_per_block(srcs[si]) : 0;
            int incl = cnt;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
            if (si < n_src) srcs[si].counts[1] = carry + incl - cnt;
            carry += __shfl_sync(0xffffffffu, incl, 31);
        }
        if (lane == 0) *total_items = carry;
    }
    __syncthreads();
    for (int si = warp; si < n_src; si += nwarps) {            // slots with a trajectory: their items, here
        Source& S = srcs[si];
        if (!has_traj(S)) continue;
        fill_traj_items(S, items, lane, 32);
        __syncwarp();
        if (lane == 0) S.counts[0] = 0;
    }
}

// ----------------------------------------------------------------------------- k_rir_absmax
// SS_RIR_NORMALIZE: partial maxima of |h| over a source's whole (P, C, L) tensor, kNormParts CTAs per source, each
// writing its own slot (no atomics, nothing to reset between runs); k_prepare's RIR rows take the maximum of the
// slots and divide their taps by it - generate_rir_combination's `ir_output /= ir_output.abs().max()`
// (SonicSim_audio.py:398) without a separate pass over the RIRs.
__global__ void __launch_bounds__(256)
k_rir_absmax(const Source* __restrict__ srcs) {
    const Source& S = srcs[blockIdx.x / kNormParts];
    if (!S.norm_part) return;
    const int part = blockIdx.x % kNormParts;
    const size_t total = (size_t)S.P * S.C * S.L;
    float m = 0.f;
    if ((((uintptr_t)S.rir) & 15) == 0) {               // 16-byte loads over the aligned bulk, scalar tail
        const float4* r4 = (const float4*)S.rir;
        const size_t n4 = total >> 2;
        for (size_t i = (size_t)part * blockDim.x + threadIdx.x; i < n4; i += (size_t)kNormParts * blockDim.x) {
            const float4 v = r4[i];
            m = fmaxf(fmaxf(m, fmaxf(fabsf(v.x), fabsf(v.y))), fmaxf(fabsf(v.z), fabsf(v.w)));
        }
        if (part == 0 && threadIdx.x < (total & 3)) m = fmaxf(m, fabsf(S.rir[(n4 << 2) + threadIdx.x]));
    } else {
        for (size_t i = (size_t)part * blockDim.x + threadIdx.x; i < total; i += (size_t)kNormParts * blockDim.x)
            m = fmaxf(m, fabsf(S.rir[i]));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    __shared__ float s_m[8];
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < 8; ++w) m = fmaxf(m, s_m[w]);
        const_cast<float*>(S.norm_part)[part] = m;
    }
}

// ----------------------------------------------------------------------------- k_rir_direct
// SS_DIRECT_TARGET: one warp per (p, c) RIR row of every direct-target source of the chunk (`per_src` CTAs of 8 rows
// per source): first-occurrence argmax of |h| over the row - on the normalised taps when the source has
// SS_RIR_NORMALIZE, so after k_rir_absmax - and the row's direct-path length cut[p, c] = min(L, peak + direct_taps),
// which k_prepare's direct rows use as their length.
__global__ void __launch_bounds__(256)
k_rir_direct(const Source* __restrict__ srcs, int per_src) {
    const Source& S = srcs[blockIdx.x / per_src];
    const int row = (blockIdx.x % per_src) * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (!S.cut || !S.rir || row >= S.P * S.C) return;          // banked source (no rir): its cut table is the bank's
    // windowed source: only the (p, c) rows its transformed RIR rows come from (the others may not even be in memory)
    if (S.h_rows && (row < S.h_row0 / S.K || row > (S.h_row0 + S.h_rows - 1) / S.K)) return;
    const float div = S.norm_part ? rir_absmax(S) : 0.f;
    PeakAt m = peak_scan(S.rir + (size_t)row * S.L, S.L, div, lane, 32);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        PeakAt q; q.v = __shfl_xor_sync(0xffffffffu, m.v, o); q.i = __shfl_xor_sync(0xffffffffu, m.i, o);
        m = peak_first(m, q);
    }
    if (lane == 0) S.cut[row] = direct_cut(m.i, S.L, S.direct_taps);
}

// ----------------------------------------------------------------------------- k_prepare
// CTA kinds, flattened per source through `prefix`:
//   [0, nh)            two RIR-partition rows  -> two half spectra (one complex FFT); a direct-target source's
//                      direct rows (length cut[p, c]) follow its reverberant ones
//   [nh, nh + nx)      two dry windows         -> two half spectra
//   [nh + nx, ...)     8 blocks each (one warp per block): position range of the block and its
//                      k_render work items (RItem)
// A CTA lives a few microseconds, so the chain of dependent loads in front of its first row load matters: for chunks of up
// to kPrepInline sources the source table and its prefix sums travel as kernel parameters (constant bank)
// instead of global memory (binary search + descriptor = 4-5 L2 round trips per CTA).
constexpr int kPrepInline = 24;
struct PrepParams {
    int n_inline;                      // 0: use the global tables
    int prefix[kPrepInline + 1];
    Source srcs[kPrepInline];
};
static_assert(sizeof(PrepParams) <= 4000, "kernel parameter space");

#ifndef SS_PREP_MINB
#define SS_PREP_MINB 2        // resident CTAs per SM the register allocation of k_prepare aims at (3 fits shared memory)
#endif
template <bool INL>
__global__ void __launch_bounds__(kThreads, SS_PREP_MINB)
k_prepare(const Source* __restrict__ srcs_g, const int* __restrict__ prefix_g, int n_src, RItem* __restrict__ items,
          const __grid_constant__ PrepParams pp) {
    extern __shared__ float2 smem[];
    const Tables T{g_tw, g_twB, g_twC};
    const int t = threadIdx.x;
    int si = 0;
    if (INL) { for (int i = 1; i < kPrepInline; ++i) si += (i < n_src && pp.prefix[i] <= (int)blockIdx.x) ? 1 : 0; }
    else si = find_source(prefix_g, n_src, blockIdx.x);
    const Source& S = INL ? pp.srcs[si] : srcs_g[si];
    int local = blockIdx.x - (INL ? pp.prefix[si] : prefix_g[si]);
    Row ra, rb;
    const int nh = spectra_pairs_h(S), nx = spectra_pairs_x(S);
    if (local >= nh + nx) {
        const int blk = (local - nh - nx) * 8 + (t >> 5), lane = t & 31;
        if (blk >= S.counts[0]) return;
        const Block bk = S.blocks[blk];
        if (S.mode == MODE_MOVING_BOUNDS && !S.aligned && blk == 0 && lane == 0) {
            // one warp per source checks the device-side bounds table
            bool bad = S.bounds[0] != 0 || S.bounds[S.P - 1] != S.N;
            for (int q = 0; q + 1 < S.P && !bad; ++q) bad = S.bounds[q + 1] < S.bounds[q];
            if (bad) atomicOr(&g_dev_err, 2u);
        }
        if ((unsigned)(blk - win_first(S)) >= (unsigned)win_blocks(S)) return;     // windowed: block outside the window
        int pmin = 0, pmax = 0;
        if (S.mode == MODE_MOVING_INDEXED) {
            block_pos_scan(S, bk, lane, 32, pmin, pmax);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                int a = __shfl_xor_sync(0xffffffffu, pmin, o), bm = __shfl_xor_sync(0xffffffffu, pmax, o);
                pmin = a < pmin ? a : pmin; pmax = bm > pmax ? bm : pmax;
            }
            // the reference raises IndexError for idx + 1 >= P (checked on the host path); block_positions clamps, leave a mark
            if (lane == 0 && (pmin < 0 || pmax + 1 > S.P - 1)) atomicOr(&g_dev_err, 1u);
        }
        fill_items(S, items, blk, block_positions(S, bk, pmin, pmax), lane, 32, stem_gain(S));
        return;
    }
    if (local < nh) rows_of_pair_h(S, local, ra, rb);
    else { local -= nh; ra = make_row_x(S, 2 * local); rb = make_row_x(S, 2 * local + 1); }
    if (!ra.dst && !rb.dst) return;              // both block slots unused (aligned blocking over-allocates)

    Regs32 R;
    spectra_phase1(t, ra, rb, smem);
    __syncthreads();
    load2(t, smem, R);
    __syncthreads();
    passB2<false>(t, smem, R, T);
    __syncthreads();
    load2(t, smem, R);
    spectra_phase3_compute(t, R, T);
    __syncthreads();
    spectra_phase3_store(t, smem, R);
    __syncthreads();
    spectra_phase4(t, smem, ra, rb);
}

// profiling aid: keeps the stream busy for `ns` nanoseconds
__global__ void k_delay(unsigned ns) {
    unsigned long long t0, t1;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
    do { __nanosleep(2000); asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1)); } while (t1 - t0 < ns);
}

// ----------------------------------------------------------------------------- k_render
// mbarrier / bulk-copy (TMA engine, 1-D) helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "LAB_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra DONE;\n"
        "bra LAB_WAIT;\n"
        "DONE:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
// work item, global -> shared, asynchronously (consumed one transform later)
__device__ __forceinline__ void item_prefetch(RItem* dst, const RItem* src) {
#pragma unroll
    for (int i = 0; i < (int)sizeof(RItem) / 16; ++i)
        asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(smem_u32((const char*)dst + 16 * i)), "l"((const char*)src + 16 * i) : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
}
__device__ __forceinline__ void item_prefetch_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

constexpr int kSpecBytes = kSpec * (int)sizeof(float2);                       // 32 KB
constexpr int kRenderSmem = kPadF * (int)sizeof(float2) + kSpecBytes;         // FFT buffer + Hq staging

#ifndef SS_RENDER_MINB
#define SS_RENDER_MINB 2
#endif
// Persistent CTAs: CTA i renders items i, i + gridDim.x, ...  Thread 0 runs one transform ahead:
// while the CTA computes transform k it has the bulk-copy engine stage transform k+1's spectra —
// Hq into the staging buffer as soon as form_z(k) has consumed it, X and Hp into the FFT buffer itself
// once pass C of transform k has read it out — so form_z never waits on L2.
// LONG: RIR partitions >= 1 are accumulated (L > 4096).  FAST: every item of the chunk is a compact-trajectory
// source under aligned blocking (one transform per block, two positions each, one segment per block).
#ifndef SS_LONG_STAGED
#define SS_LONG_STAGED 1          // 0: partitions >= 1 read with plain loads (form_z_parts), for comparison
#endif
template <bool LONG, bool FAST>
__global__ void __launch_bounds__(kThreads, SS_RENDER_MINB)
k_render(const RItem* __restrict__ items, const int* __restrict__ n_items_ptr, int n_items_host) {
    extern __shared__ __align__(128) float2 smem[];
    __shared__ __align__(16) RItem s_item[2];
    __shared__ __align__(16) XDesc s_desc[2];
    __shared__ __align__(8) uint64_t s_bar[2];          // [0]: X + Hp landed, [1]: Hq landed
    float2* const fftbuf = smem;
    float2* const sX = smem;
    float2* const sHp = smem + kSpec;
    float2* const sHq = smem + kPadF;
    const Tables T{g_tw, g_twB, g_twC};
    const int t = threadIdx.x;
    // table length: known on the host when it built the tables, otherwise written by k_blocks
    const int n_items = n_items_host >= 0 ? n_items_host : *n_items_ptr;

    // thread-0 iterator state
    int it_cur = blockIdx.x;          // item of the transform most recently published
    int slot = 0;                     // s_item slot holding it
    int p_cur = 0;

    if (t == 0) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        XDesc d; d.valid = 0; d.Hq = nullptr;
        if (it_cur < n_items) {
            s_item[0] = items[it_cur];
            if (it_cur + (int)gridDim.x < n_items) item_prefetch(&s_item[1], &items[it_cur + gridDim.x]);
            p_cur = s_item[0].p_lo;
            d = make_xdesc(s_item[0], p_cur);
        }
        s_desc[0] = d;
        fence_proxy_async();
        if (d.valid) {
            mbar_expect_tx(&s_bar[0], 2 * kSpecBytes);
            bulk_g2s(sX, d.X, kSpecBytes, &s_bar[0]);
            bulk_g2s(sHp, d.Hp, kSpecBytes, &s_bar[0]);
            if (d.Hq) { mbar_expect_tx(&s_bar[1], kSpecBytes); bulk_g2s(sHq, d.Hq, kSpecBytes, &s_bar[1]); }
            else mbar_arrive(&s_bar[1]);
        } else { mbar_arrive(&s_bar[0]); mbar_arrive(&s_bar[1]); }
    }
    __syncthreads();

    Regs32 R;
    unsigned ph = 0;                                  // parity of the staging barriers' current phase
    for (int k = 0;; ++k) {
        mbar_wait(&s_bar[0], ph);
        mbar_wait(&s_bar[1], ph);
        ph ^= 1;
        const XDesc& d = s_desc[k & 1];
        if (!d.valid) break;
        if (LONG && SS_LONG_STAGED) {
            // partitions 1 .. kparts-1 follow partition 0 through the same staging buffers
            const float2* const q = d.Hq ? sHq : nullptr;
            DcNy e;
            long_stage<true>(t, sX, sHp, q, R, e);
            const int kparts = d.kparts;
            for (int part = 1; part < kparts; ++part) {
                __syncthreads();                      // partition part-1 consumed by every thread
                if (t == 0) {
                    fence_proxy_async();
                    mbar_expect_tx(&s_bar[0], 2 * kSpecBytes);
                    bulk_g2s(sX, d.X - (size_t)part * kSpec, kSpecBytes, &s_bar[0]);
                    bulk_g2s(sHp, d.Hp + (size_t)part * kSpec, kSpecBytes, &s_bar[0]);
                    if (d.Hq) { mbar_expect_tx(&s_bar[1], kSpecBytes); bulk_g2s(sHq, d.Hq + (size_t)part * kSpec, kSpecBytes, &s_bar[1]); }
                    else mbar_arrive(&s_bar[1]);
                }
                mbar_wait(&s_bar[0], ph);
                mbar_wait(&s_bar[1], ph);
                ph ^= 1;
                long_stage<false>(t, sX, sHp, q, R, e);
            }
            long_finish(t, R, e);
        } else {
            form_z<LONG, FAST>(t, sX, sHp, (FAST || d.Hq) ? sHq : nullptr, d, R);
        }
        __syncthreads();                              // staged spectra consumed, s_desc[k & 1] read by all
        if (t == 0) {
            // publish transform k+1 and start staging its Hq
            XDesc nx; nx.valid = 0; nx.Hq = nullptr;
            const RItem& cur = s_item[slot];
            if (p_cur + 2 <= cur.p_hi) { p_cur += 2; nx = make_xdesc(cur, p_cur); }
            else if (it_cur + (int)gridDim.x < n_items) {
                it_cur += gridDim.x; slot ^= 1;
                item_prefetch_wait();                 // issued one item ago
                p_cur = s_item[slot].p_lo;
                nx = make_xdesc(s_item[slot], p_cur);
                if (it_cur + (int)gridDim.x < n_items) item_prefetch(&s_item[slot ^ 1], &items[it_cur + gridDim.x]);
            }
            s_desc[(k + 1) & 1] = nx;
            fence_proxy_async();
            if (nx.valid && nx.Hq) { mbar_expect_tx(&s_bar[1], kSpecBytes); bulk_g2s(sHq, nx.Hq, kSpecBytes, &s_bar[1]); }
            else mbar_arrive(&s_bar[1]);
        }
        render_phase1(t, fftbuf, R);
        __syncthreads();
        load2(t, fftbuf, R);
        __syncthreads();
        passB2<true>(t, fftbuf, R, T);
        __syncthreads();
        load2(t, fftbuf, R);
        __syncthreads();                              // FFT buffer is free: stage X, Hp of transform k+1 into it
        if (t == 0) {
            const XDesc nx = s_desc[(k + 1) & 1];
            fence_proxy_async();
            if (nx.valid) {
                mbar_expect_tx(&s_bar[0], 2 * kSpecBytes);
                bulk_g2s(sX, nx.X, kSpecBytes, &s_bar[0]);
                bulk_g2s(sHp, nx.Hp, kSpecBytes, &s_bar[0]);
            } else mbar_arrive(&s_bar[0]);
        }
        render_phase3(t, R, T);
        render_epilogue<FAST>(t, d, R);
    }
}

// ----------------------------------------------------------------------------- k_render_fast
// Chunks whose items are one transform each: compact trajectories under aligned blocking (the transform packs the
// positions (s, s + 1) of the block's segment) and static sources (two channels per transform), L <= 4096: every source
// of BASELINE configs[1] / [2] and of a SonicSet scene.  Same phases as k_render; what differs is who
// feeds the bulk-copy engine and how many bytes pass through the SM's L1 / shared-memory data pipe, which together with
// the issue slots is what the kernel runs against (DESIGN.md section 4, profiles/EXPERIMENTS.md):
//   * a CTA renders a CONTIGUOUS range of items: the channels of a block are neighbours and share the dry spectrum X,
//     which lives in its own 32 KB buffer and is copied only when the next item belongs to another block (one lane
//     of warp 7, right after the staged spectra have been consumed);
//   * the filter spectra Hp, Hq of the next transform land in the FFT buffer itself; their copy is issued by whichever
//     warp is the LAST to finish its pass-C loads (a shared counter tells), so nobody waits for the buffer to drain;
//   * no serial producer section: work items are final (k_prepare wrote pointers, sample range, segment start and
//     1 / length) and prefetched two transforms ahead with cp.async;
//   * inter-pass twiddles: 4 table rows + 11 products per pass (tw_get) instead of 15 loads.
// Measured and rejected (profiles/EXPERIMENTS.md, profiles/r2_exp_fast_knobs.patch): split arrive / wait mbarriers
// instead of two of the four CTA barriers, twiddle loads hoisted above the exchange barriers, twiddles from registers
// only, a fixed producer lane waiting for the buffer - none of them moves the kernel.
constexpr int kItemLane = 7 * 32;     // thread that prefetches work items and issues the X copies (not warp 0, whose
                                      // thread 0 already carries the DC / Nyquist words)
__device__ __forceinline__ unsigned atom_inc_acqrel(unsigned* p) {
    unsigned old;
    asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], 1;" : "=r"(old) : "r"(smem_u32(p)) : "memory");
    return old;
}
// both butterflies of a thread, the 16 loads of butterfly t first so that its arithmetic can start while the
// loads of butterfly t + 256 are still in flight
__device__ __forceinline__ void load2_ab(int t, const float2* s, Regs32& R) {
    const float2* p = s + pad(t);
#pragma unroll
    for (int r = 0; r < 16; ++r) R.a[r] = p[544 * r];
#pragma unroll
    for (int r = 0; r < 16; ++r) R.b[r] = p[544 * r + 272];
}
template <bool GAIN>
__global__ void __launch_bounds__(kThreads, SS_RENDER_MINB)
k_render_fast(const RItem* __restrict__ items, const int* __restrict__ n_items_ptr, int n_items_host) {
    extern __shared__ __align__(128) float2 smem[];
    __shared__ __align__(16) RItem s_item[3];
    __shared__ __align__(8) uint64_t s_bar[2];          // [0] Hp + Hq landed, [1] X landed or kept (transaction counts)
    __shared__ unsigned s_drained;                      // warps that have finished their pass-C loads, cumulative
    float2* const fftbuf = smem;
    float2* const sHp = smem;                           // the filter spectra land in the FFT buffer itself
    float2* const sHq = smem + kSpec;
    float2* const sX = smem + kPadF;                    // the dry spectrum has its own buffer: it survives the transform
    const Tables T{g_tw, g_twB, g_twC};
    const int t = threadIdx.x, lane = t & 31;
    // table length: known on the host when it built the tables, otherwise written by k_blocks
    const int n_items = n_items_host >= 0 ? n_items_host : *n_items_ptr;
    const int per = n_items / (int)gridDim.x, rem = n_items % (int)gridDim.x;
    const int n_k = per + ((int)blockIdx.x < rem ? 1 : 0);              // transforms of this CTA: a contiguous range
    if (n_k <= 0) return;
    const RItem* const my_items = items + (size_t)blockIdx.x * per + ((int)blockIdx.x < rem ? (int)blockIdx.x : rem);

    if (t == kItemLane) {
        mbar_init(&s_bar[0], 1);
        mbar_init(&s_bar[1], 1);
        s_drained = 0;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        s_item[0] = my_items[0];
        if (n_k > 1) s_item[1] = my_items[1];
        fence_proxy_async();
        mbar_expect_tx(&s_bar[0], 2 * kSpecBytes);
        bulk_g2s(sHp, item_hp(s_item[0]), kSpecBytes, &s_bar[0]);
        bulk_g2s(sHq, item_hq(s_item[0]), kSpecBytes, &s_bar[0]);
        mbar_expect_tx(&s_bar[1], kSpecBytes);
        bulk_g2s(sX, s_item[0].X, kSpecBytes, &s_bar[1]);
    }
    __syncthreads();

    Regs32 R;
    float2 w[16];
    XDesc unused; unused.kparts = 1; unused.Hq = nullptr; unused.X = nullptr; unused.Hp = nullptr;
    unsigned ph = 0;
    for (int k = 0; k < n_k; ++k) {
        mbar_wait(&s_bar[0], ph);
        mbar_wait(&s_bar[1], ph);
        form_z<false, true>(t, sX, sHp, sHq, unused, R);
        fft16<true>(R.a);
        fft16<true>(R.b);
        __syncthreads();                                  // B1: staged spectra consumed, pass A may overwrite Hp / Hq
        if (t == kItemLane) {
            if (k + 1 < n_k) {                            // item k + 1 became visible at barrier B4 of transform k - 1
                const RItem& nx = s_item[(k + 1) % 3];
                if (nx.X != s_item[k % 3].X) {            // next item belongs to another block: its dry spectrum
                    fence_proxy_async();
                    mbar_expect_tx(&s_bar[1], kSpecBytes);
                    bulk_g2s(sX, nx.X, kSpecBytes, &s_bar[1]);
                } else mbar_arrive(&s_bar[1]);            // same block, other channel: X stays where it is
            }
            // item k + 2 into the slot of item k - 1 (last read in the output stage of k - 1, which every warp has left)
            if (k + 2 < n_k) item_prefetch(&s_item[(k + 2) % 3], my_items + (k + 2));
        }
        passA_store(fftbuf, passA_jA(t), R.a);
        passA_store(fftbuf, passA_jB(t), R.b);
        __syncthreads();                                  // B2: pass A -> pass B exchange
        load2_ab(t, fftbuf, R);
        tw_get<true, 16>(T.twB + (t & 15), w);
        fft16_w<true>(R.a, w);
        fft16_w<true>(R.b, w);
        __syncthreads();                                  // B3: every warp has loaded its pass-B inputs
        passB_store(fftbuf, t, R.a);
        passB_store(fftbuf, t + 256, R.b);
        if (t == kItemLane) item_prefetch_wait();         // item k + 2 has landed; visible to all behind B4
        __syncthreads();                                  // B4: pass B -> pass C exchange
        load2_ab(t, fftbuf, R);
        tw_get<true, 256>(T.twC + t, w);
        __syncwarp();
        if (lane == 0 && atom_inc_acqrel(&s_drained) == (unsigned)(8 * k + 7) && k + 1 < n_k) {
            // last warp out of the FFT buffer: stage Hp, Hq of transform k + 1 into it
            const RItem& nx = s_item[(k + 1) % 3];
            fence_proxy_async();
            mbar_expect_tx(&s_bar[0], 2 * kSpecBytes);
            bulk_g2s(sHp, item_hp(nx), kSpecBytes, &s_bar[0]);
            bulk_g2s(sHq, item_hq(nx), kSpecBytes, &s_bar[0]);
        }
        ph ^= 1;
        fft16_w<true>(R.a, w);                            // pass C
        fft16_w<true>(R.b, w);
        render_phase3_close(t, R, T);
        render_epilogue_item<GAIN>(t, s_item[k % 3], R);
    }
}

// ============================================================================= host side
thread_local int g_last_cuda = 0;

extern "C" int ss_version(void) { return 108; }
extern "C" int ss_last_cuda_error(void) { return g_last_cuda; }
extern "C" const char* ss_strerror(int st) {
    switch (st) {
        case SS_OK: return "ok";
        case SS_ERR_INVALID: return "invalid argument";
        case SS_ERR_INDEX: return "index out of bounds: trajectory refers to position >= P - 1";
        case SS_ERR_CUDA: return "CUDA runtime error";
        case SS_ERR_NOMEM: return "out of device / pinned memory";
        case SS_ERR_UNSUPPORTED: return "unsupported shape";
        default: return "unknown status";
    }
}


extern "C" void ss_destroy(ss_ctx* c);

static int init_ctx(ss_ctx* c, int device) {
    CK(cudaSetDevice(device));
    c->device = device;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    c->sm_count = prop.multiProcessorCount;
    std::vector<float2> tw(kF);
    for (int m = 0; m < kF; ++m) {
        double a = -2.0 * M_PI * (double)m / (double)kF;
        tw[m] = make_float2((float)cos(a), (float)sin(a));
    }
    CK(cudaMemcpyToSymbol(g_tw, tw.data(), sizeof(float2) * kF));
    std::vector<float2> tb(kTabB), tc(kTabC);
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
    CK(cudaMemcpyToSymbol(g_twB, tb.data(), sizeof(float2) * kTabB));
    CK(cudaMemcpyToSymbol(g_twC, tc.data(), sizeof(float2) * kTabC));
    { const unsigned zero = 0; CK(cudaMemcpyToSymbol(g_dev_err, &zero, sizeof(zero))); }
    CK(cudaFuncSetAttribute(k_prepare<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPadF * (int)sizeof(float2)));
    CK(cudaFuncSetAttribute(k_prepare<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kPadF * (int)sizeof(float2)));
    CK(cudaFuncSetAttribute(k_render<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmem));
    CK(cudaFuncSetAttribute(k_render_fast<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmem));
    CK(cudaFuncSetAttribute(k_render_fast<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmem));
    CK(cudaFuncSetAttribute(k_render<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmem));
    for (int i = 0; i < ss_ctx::kRing; ++i) {
        CK(cudaEventCreateWithFlags(&c->desc_ev[i], cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->desc_done[i], cudaEventDisableTiming));
    }
    for (int i = 0; i < ss_ctx::kAux; ++i) {
        CK(cudaStreamCreateWithFlags(&c->s_aux[i], cudaStreamNonBlocking));
        CK(cudaEventCreateWithFlags(&c->ev_join[i], cudaEventDisableTiming));
    }
    CK(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
    CK(cudaStreamCreateWithFlags(&c->s_in, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->s_cmp, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&c->s_out, cudaStreamNonBlocking));
    for (int i = 0; i < ss_ctx::kSlots; ++i) {
        CK(cudaEventCreateWithFlags(&c->slot[i].ev_in, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->slot[i].ev_done, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->slot[i].ev_rend, cudaEventDisableTiming));
        CK(cudaEventCreateWithFlags(&c->slot[i].ev_free, cudaEventDisableTiming));
    }
    c->single_stream = getenv("SS_SINGLE_STREAM") != nullptr;
    c->no_fast = getenv("SS_NO_FAST") != nullptr;
    c->no_graph = getenv("SS_NO_GRAPH") != nullptr;
    if (getenv("SS_HOST_CHUNK_MB")) c->chunk_bytes_host = (int64_t)atoi(getenv("SS_HOST_CHUNK_MB")) << 20;
    return SS_OK;
}

extern "C" int ss_create(int device, ss_ctx** out) {
    if (!out) return SS_ERR_INVALID;
    *out = nullptr;
    ss_ctx* c = new (std::nothrow) ss_ctx();
    if (!c) return SS_ERR_NOMEM;
    const int st = init_ctx(c, device);
    if (st != SS_OK) { ss_destroy(c); return st; }        // releases whatever was created before the failure
    *out = c;
    return SS_OK;
}

extern "C" void ss_destroy(ss_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    for (int i = 0; i < ss_ctx::kAux; ++i) {
        if (c->d_scratch[i]) cudaFree(c->d_scratch[i]);
        if (c->s_aux[i]) cudaStreamDestroy(c->s_aux[i]);
        if (c->ev_join[i]) cudaEventDestroy(c->ev_join[i]);
    }
    if (c->ev_fork) cudaEventDestroy(c->ev_fork);
    for (int i = 0; i < ss_ctx::kRing; ++i) {
        if (c->h_desc[i]) cudaFreeHost(c->h_desc[i]);
        if (c->d_desc[i]) cudaFree(c->d_desc[i]);
        if (c->desc_ev[i]) cudaEventDestroy(c->desc_ev[i]);
        if (c->desc_done[i]) cudaEventDestroy(c->desc_done[i]);
    }
    for (int i = 0; i < ss_ctx::kSlots; ++i) {
        if (c->slot[i].d_in) cudaFree(c->slot[i].d_in);
        if (c->slot[i].d_out) cudaFree(c->slot[i].d_out);
        if (c->slot[i].ev_in) cudaEventDestroy(c->slot[i].ev_in);
        if (c->slot[i].ev_done) cudaEventDestroy(c->slot[i].ev_done);
        if (c->slot[i].ev_rend) cudaEventDestroy(c->slot[i].ev_rend);
        if (c->slot[i].ev_free) cudaEventDestroy(c->slot[i].ev_free);
    }
    if (c->h_post) cudaFreeHost(c->h_post);
    if (c->d_post) cudaFree(c->d_post);
    if (c->s_in) cudaStreamDestroy(c->s_in);
    if (c->s_cmp) cudaStreamDestroy(c->s_cmp);
    if (c->s_out) cudaStreamDestroy(c->s_out);
    delete c;
}

// Bits set by the kernels of this context's device since the last call (waits for the device to go idle).
extern "C" int ss_device_errors(ss_ctx* c, uint32_t* bits) {
    if (!c || !bits) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    CK(cudaDeviceSynchronize());
    unsigned v = 0, zero = 0;
    CK(cudaMemcpyFromSymbol(&v, g_dev_err, sizeof(v)));
    if (v) CK(cudaMemcpyToSymbol(g_dev_err, &zero, sizeof(zero)));
    *bits = v;
    return SS_OK;
}

extern "C" int ss_set_chunk_bytes(ss_ctx* c, int64_t bytes) {
    if (!c || bytes < (1 << 20)) return SS_ERR_INVALID;
    c->chunk_bytes = bytes;
    return SS_OK;
}
extern "C" int64_t ss_launch_count(const ss_ctx* c) { return c ? c->launches : 0; }
extern "C" void ss_reset_stats(ss_ctx* c) { if (c) c->launches = 0; }

extern "C" int ss_set_profiling(ss_ctx* c, int on) {
    if (!c) return SS_ERR_INVALID;
    c->profiling = on != 0;
    return SS_OK;
}
// Sum of per-launch device times since the last call (waits for the recorded work to finish).
extern "C" int ss_get_profile(ss_ctx* c, double* ms_spectra, double* ms_render, int64_t* n_pairs) {
    if (!c) return SS_ERR_INVALID;
    // Launch pairs with the same position inside their render call repeat the same work: each group contributes
    // (median over the calls) x (group size), so a host hiccup that leaves the GPU waiting inside one interval
    // does not leak into the sums.
    std::vector<std::vector<float>> ta, tb;
    for (auto& pf : c->prof) {
        CK(cudaEventSynchronize(pf.e2));
        float t1 = 0, t2 = 0;
        CK(cudaEventElapsedTime(&t1, pf.e0, pf.e1));
        CK(cudaEventElapsedTime(&t2, pf.e1, pf.e2));
        if ((size_t)pf.chunk >= ta.size()) { ta.resize(pf.chunk + 1); tb.resize(pf.chunk + 1); }
        ta[pf.chunk].push_back(t1); tb[pf.chunk].push_back(t2);
        cudaEventDestroy(pf.e0); cudaEventDestroy(pf.e1); cudaEventDestroy(pf.e2);
    }
    auto robust_sum = [](std::vector<std::vector<float>>& groups) {
        double s = 0;
        for (auto& g : groups) {
            if (g.empty()) continue;
            std::sort(g.begin(), g.end());
            const size_t n = g.size();
            const double med = (n & 1) ? g[n / 2] : 0.5 * ((double)g[n / 2 - 1] + g[n / 2]);
            s += med * (double)n;
        }
        return s;
    };
    const double a = robust_sum(ta), b = robust_sum(tb);
    if (ms_spectra) *ms_spectra = a;
    if (ms_render) *ms_render = b;
    if (n_pairs) *n_pairs = (int64_t)c->prof.size();
    c->prof.clear();
    return SS_OK;
}

extern "C" int ss_host_alloc(void** p, int64_t bytes) {
    if (!p || bytes <= 0) return SS_ERR_INVALID;
    CK(cudaHostAlloc(p, (size_t)bytes, cudaHostAllocDefault));
    return SS_OK;
}
extern "C" void ss_host_free(void* p) { if (p) cudaFreeHost(p); }

// RIR spectrum bank: one device allocation = [reverberant set | direct set] (P*C*K rows of kSpec float2 each, the layout
// k_prepare writes into chunk scratch) | cut table (direct set) | descriptor of the blockless source that built it |
// its norm_part slots (SS_RIR_NORMALIZE).  A host bank's block (SS_BANK_HOST) is [spectra | cut table], unpadded; a
// tap-form host bank (SS_BANK_TAPS) holds the padded tap rows (tap_value) in place of the spectra, in both places.
struct ss_bank {
    ss_ctx* c = nullptr;                  // the context that made it; sources of other contexts are refused
    char* d_mem = nullptr;
    size_t bytes = 0;
    float2* spec = nullptr;
    int* cut = nullptr;                   // P*C direct-path row lengths, or null: no direct set
    int P = 0, C = 0, L = 0, K = 0, flags = 0, direct_taps = 0;
    cudaEvent_t ready = nullptr;          // recorded behind the launches that build it; every use waits on it
    // SS_BANK_HOST: spectra and cut table moved into pinned, mapped host memory (spec / cut: their device addresses)
    char* h_mem = nullptr;
    size_t host_bytes = 0;
    // bytes of one set of spectra, of every set, and of the cut table, which follows the spectra in both layouts
    size_t set_bytes() const { return (size_t)P * C * K * kSpec * sizeof(float2); }
    size_t spec_bytes() const { return ((flags & SS_DIRECT_TARGET) ? 2 : 1) * set_bytes(); }
    size_t cut_bytes() const { return (flags & SS_DIRECT_TARGET) ? sizeof(int) * (size_t)P * C : 0; }
    // SS_BANK_TAPS: the P*C*K rows of kB taps, one set whatever the flags (`spec` then holds their address)
    size_t tap_bytes() const { return (size_t)P * C * K * kB * sizeof(float); }
    size_t head_bytes() const { return (flags & SS_BANK_TAPS) ? tap_bytes() : spec_bytes(); }   // in front of the cuts
};
// Source pool: the candidates' compact entries in one device allocation, and on the host what validation, sizing and the
// mixture range checks need.
struct ss_pool {
    ss_ctx* c = nullptr;
    PoolEntry* table = nullptr;           // device, n entries
    int n = 0, mode = 0, C = 0, L = 0, K = 0, aligned = 0;   // L, K: the longest candidate's
    std::vector<int> parts_host;          // candidate i's RIR partition count K_i
    int* parts = nullptr;                 // device copy of parts_host when the K_i differ (pool_parts), else null
    int n_min = 0, p_max = 0;             // shortest candidate (window rule), most positions (rstep table)
    int direct_taps = 0;                  // > 0: every candidate's bank holds a direct set with these taps
    std::vector<PoolEntry> host;          // the table's entries
    std::vector<int32_t> bounds_host;     // every moving candidate's bounds, back to back
    std::vector<int64_t> bounds_off;      // candidate i's bounds at bounds_host[bounds_off[i]]
    std::vector<std::pair<int, int>> caps;  // (win_len, table size) already worked out (pool_table_cap)
    std::vector<std::pair<int, int>> traj_caps;   // the same for slots with a trajectory (traj_table_cap)
    std::vector<const ss_bank*> banks;    // candidate i's bank (ss_pool_levels renders the candidates)
    cudaEvent_t ready = nullptr;          // behind the construction of every candidate's bank
    // level tables (ss_pool_levels): every candidate's N + 1 doubles back to back, and a device array of n pointers
    double* levels = nullptr;
    double* h_levels = nullptr;           // a host pool's tables: their host address (levels: their device address)
    const double** level_ptr = nullptr;
    std::vector<int64_t> level_off;       // candidate i's table at levels + level_off[i]
    int level_flags = -1;                 // SS_MIX_MONO or 0 once the tables exist
    // loudness gains (ss_pool_loudness): n floats (float)gain on the device, 1 for an unmeasured candidate, and the
    // measured (LUFS, gain) pairs on the host
    float* gains = nullptr;
    std::vector<double> loud;
    bool planned = false;                 // a plan has been created over the pool: its gains may no longer change
    // host pool (every candidate's bank has SS_BANK_HOST): x in one pinned, mapped arena (host[i].x: its device address);
    // the device copies of the bounds and cut tables in one device allocation (host[i].bounds / cut point into it)
    bool host_res = false;
    bool taps = false;                    // a host pool of tap-form banks (SS_BANK_TAPS): entries' spec hold tap rows
    char* h_x = nullptr;
    size_t h_x_bytes = 0;
    int* d_aux = nullptr;
    size_t aux_bytes = 0;
    std::vector<std::pair<int, std::pair<int, int>>> stage_caps;  // (win_len, (rows, dry samples)) (stage_cap)
};
// Dry pool: n dry signals referenced by their device pointers (the caller's buffers), the device array of those pointers
// that dry-picked slots index (dry_table), and with SS_DRY_LEVELS every signal's level table.  A host dry pool
// (SS_DRY_HOST) owns its signals, copied into one pinned, mapped arena, and keeps its tables in pinned, mapped host
// memory: x, ptrs, levels and level_ptr then hold mapped device addresses.
// A 16-bit dry pool (ss_dry_pool_create_i16) owns one arena of int16 signals, in device memory or (SS_DRY_HOST) pinned,
// mapped host memory; ptrs and x16 hold int16 addresses, x is empty, and its tables are sparse (kLevelStride): signal
// i's ceil(N / 64) + 1 entries at levels + level_off[i].  With tables, ptrs holds 2n pointers, the n signals' and then
// the n tables' (level_ptr = ptrs + n, not allocated on its own), which k_draw reads both of (speaker_signal_i16).
struct ss_dry_pool {
    ss_ctx* c = nullptr;
    int n = 0, n_min = 0;                 // n_min: the shortest signal (the longest candidate N it serves)
    const float** ptrs = nullptr;         // device, n signal pointers
    std::vector<const float*> x;          // the same pointers on the host
    std::vector<int32_t> N;
    double* levels = nullptr;             // device: every signal's N + 1 doubles back to back
    const double** level_ptr = nullptr;   // device, n table pointers
    std::vector<int64_t> level_off;       // signal i's table at levels + level_off[i]
    bool host = false;                    // SS_DRY_HOST
    char* h_x = nullptr;                  // the arena (host address) and its bytes
    size_t h_x_bytes = 0;
    double* h_levels = nullptr;           // the tables' host address
    bool i16 = false;                     // a 16-bit pool ...
    std::vector<const int16_t*> x16;      // ... its signals' device (or mapped) addresses ...
    char* d_x = nullptr;                  // ... and its device arena and its bytes (without SS_DRY_HOST)
    size_t d_x_bytes = 0;
    int stride() const { return i16 ? kLevelStride : 1; }
    bool padded() const { return host || i16; }   // owns an arena padded for k_stage's wide loads
};
// Order `stream` after the construction of every bank the items use (a bank built from device memory is built
// asynchronously on its creator's stream, which a render may not share: the host path runs on the context's own streams).
static int wait_banks(const ss_source* items, int n, cudaStream_t stream) {
    const ss_bank* last = nullptr;
    for (int i = 0; i < n; ++i) {
        const ss_bank* b = items[i].rir_bank;
        if (!b || b == last) continue;                  // (one wait per run of sources sharing a bank)
        CK(cudaStreamWaitEvent(stream, b->ready, 0));
        last = b;
    }
    return SS_OK;
}

// A banked source against its bank (include/sonicsim_b200.h): same shape, normalisation left to the bank, a direct
// target only with the bank's direct set and taps.  (A static source has P == 1 and a moving one P >= 2, checked by
// validate_item, so the shape check also gives the bank's P the source's mode.)
static int bank_fits(const ss_source& it) {
    const ss_bank* b = it.rir_bank;
    if (it.P != b->P || it.C != b->C || it.L != b->L) return SS_ERR_INVALID;
    if (it.flags & SS_RIR_NORMALIZE) return SS_ERR_INVALID;
    if ((it.flags & SS_DIRECT_TARGET) && (!b->cut || it.direct_taps != b->direct_taps)) return SS_ERR_INVALID;
    return SS_OK;
}
// a source rendered from a bank: a host bank (SS_BANK_HOST) serves only as a candidate of a host pool
static int validate_bank_use(const ss_source& it) { return it.rir_bank->h_mem ? SS_ERR_INVALID : bank_fits(it); }
static int validate_item(const ss_source& it) {
    if (it.pool || it.pick_dev) return SS_ERR_INVALID;              // pooled slots: plans only (validate_pooled)
    if (!it.x || !it.out || (it.rir != nullptr) == (it.rir_bank != nullptr)) return SS_ERR_INVALID;   // rir xor bank
    if (it.N <= 0 || it.C <= 0 || it.L <= 0 || it.P <= 0) return SS_ERR_INVALID;
    // 32-bit sample / table indices inside the kernels: leave one FFT of headroom below 2^31
    if (it.N > 0x7fffffff - 2 * kF) return SS_ERR_UNSUPPORTED;
    if ((int64_t)it.P * it.C * ((it.L + kB - 1) / kB) > (int64_t)1 << 28) return SS_ERR_UNSUPPORTED;
    if (it.flags & ~(SS_RIR_NORMALIZE | SS_DIRECT_TARGET)) return SS_ERR_INVALID;
    if ((it.flags & SS_DIRECT_TARGET) && (!it.out_direct || it.direct_taps < 1 || it.out_direct == it.out))
        return SS_ERR_INVALID;
    if (it.mode == SS_STATIC) { if (it.P != 1) return SS_ERR_INVALID; }
    else if (it.mode == SS_MOVING_BOUNDS) { if (it.P < 2 || !it.bounds) return SS_ERR_INVALID; }
    else if (it.mode == SS_MOVING_INDEXED) { if (it.P < 2 || !it.idx || !it.w) return SS_ERR_INVALID; }
    else return SS_ERR_INVALID;
    if (it.win_len < 0 || it.win_start < 0 || (it.win_len == 0 && it.win_start != 0) ||
        (int64_t)it.win_start + it.win_len > (int64_t)it.N)
        return SS_ERR_INVALID;
    // a moving window: a length, no host start, an int32 the kernels can load
    if (it.win_start_dev && (it.win_len == 0 || it.win_start != 0 || ((uintptr_t)it.win_start_dev & 3)))
        return SS_ERR_INVALID;
    return it.rir_bank ? validate_bank_use(it) : SS_OK;
}
// every bank of a batch belongs to the context that renders it
static int validate_item_ctx(const ss_ctx* c, const ss_source& it) {
    const int st = validate_item(it);
    if (st) return st;
    return (it.rir_bank && it.rir_bank->c != c) ? SS_ERR_INVALID : SS_OK;
}
// A trajectory bounds table as the header requires it: ascending from 0 to N.  Checked before anything plans blocks from
// it - a table outside the contract would make the host-side block planner write past the table it sized.
static bool bounds_ok(const int32_t* b, int P, int N) {
    if (b[0] != 0 || b[P - 1] != N) return false;
    for (int q = 0; q + 1 < P; ++q) if (b[q + 1] < b[q]) return false;
    return true;
}
// A pooled slot against its pool (include/sonicsim_b200.h): no source fields of its own, the pool's mode / C / L (the
// longest candidate's), a
// window every candidate holds, a direct target only when every candidate's bank has the slot's direct set.
static int validate_pooled(const ss_ctx* c, const ss_source& it) {
    const ss_pool* pl = it.pool;
    if (pl->c != c || !it.pick_dev || ((uintptr_t)it.pick_dev & 3) || !it.out) return SS_ERR_INVALID;
    if (it.x || it.rir || it.rir_bank || it.bounds || it.bounds_host || it.idx || it.w || it.N || it.P)
        return SS_ERR_INVALID;
    if (it.mode != pl->mode || it.C != pl->C || it.L != pl->L) return SS_ERR_INVALID;
    if (it.win_len <= 0 || it.win_start < 0 || (int64_t)it.win_start + it.win_len > (int64_t)pl->n_min)
        return SS_ERR_INVALID;
    if (it.win_start_dev && (it.win_start != 0 || ((uintptr_t)it.win_start_dev & 3))) return SS_ERR_INVALID;
    if (it.flags & ~SS_DIRECT_TARGET) return SS_ERR_INVALID;
    if ((it.flags & SS_DIRECT_TARGET) && (!it.out_direct || it.out_direct == it.out || it.direct_taps < 1 ||
                                          it.direct_taps != pl->direct_taps))
        return SS_ERR_INVALID;
    return SS_OK;
}
// SS_DIRECT_TARGET: a second RIR set (spectra, items per block) and the P*C cut table
static int direct_sets(const ss_source& it) { return (it.flags & SS_DIRECT_TARGET) ? 2 : 1; }
// spectra and cuts in a bank (a pooled slot's: in its candidates' banks), not in the chunk's scratch
static bool banked(const ss_source& it) { return it.rir_bank || it.pool; }
// RIR sets and cut table in the chunk's scratch: none for a banked source, whose spectra and cuts live in its bank
static int scratch_sets(const ss_source& it) { return banked(it) ? 0 : direct_sets(it); }
static size_t cut_bytes(const ss_source& it) {
    return ((it.flags & SS_DIRECT_TARGET) && !banked(it)) ? align_up(sizeof(int) * (size_t)it.P * it.C, 256) : 0;
}
// shapes derived from one ss_source
struct Shape {
    int K, nb, aligned, nblk_max, per, max_items;
    int p_max;                // rstep entries: P, or the largest candidate's P for a pooled slot
    // time window (win_len > 0); zero otherwise
    int win;
    int pooled;               // a pooled slot (shape_pooled)
    int traj;                 // a pooled slot with a trajectory (ss_trajectory): tables sized by traj_table_cap
    int tab_host;             // the window's blocks are known here (all but aligned blocking over device-side bounds)
    int g0, g1, k0, k1;       // tab_host: full-table blocks in the table / meeting the window (window_span)
    int row0, rows;           // RIR rows transformed per set (window_rows)
    int pa, pb;               // RIR positions read: [pa, pb]
    int xa, xb;               // dry samples read: [xa, xb)
    int ia, ib;               // idx / w entries read: [ia, ib)
};
// Aligned blocking costs one transform per block, sum_s ceil(n_s / 4096); grid blocking costs
// ceil(positions touched / 2) per 4096-block.  With the bounds on the host both counts are exact and the
// cheaper plan wins (trajectories with many short segments are better off on the grid); without them the
// plan is aligned when the average segment is at least one block long.
static bool choose_aligned(const ss_source& it, int K, int nb) {
    if (it.mode != SS_MOVING_BOUNDS || K != 1) return false;
    const int32_t* hb = it.bounds_host;
    if (!hb) return (int64_t)(it.P - 1) * kB <= (int64_t)it.N;
    int64_t aligned = 0, grid = 0;
    for (int sg = 0; sg + 1 < it.P; ++sg) aligned += seg_blocks(hb[sg + 1] - hb[sg]);
    int lo = 0;                                          // first segment that reaches into the current block
    for (int b = 0; b < nb; ++b) {
        const int n0 = b * kB, n1 = (n0 + kB < it.N ? n0 + kB : it.N) - 1;
        while (lo + 2 < it.P && hb[lo + 1] <= n0) ++lo;
        int hi = lo;
        while (hi + 2 < it.P && hb[hi + 1] <= n1) ++hi;
        grid += (hi - lo + 2 + 1) / 2;                   // positions lo .. hi + 1, two per transform
    }
    return aligned <= grid;
}
// Window of a windowed source: which blocks, RIR rows, dry samples and trajectory entries it uses (its read set, see
// include/sonicsim_b200.h).  The blocking itself is the full source's (choose_aligned over the whole trajectory).
static void window_shape(const ss_source& it, Shape& s) {
    const int ws = it.win_start, we = it.win_start + it.win_len;
    const int32_t* hb = it.mode == SS_MOVING_BOUNDS ? it.bounds_host : nullptr;
    s.win = 1;
    if (it.win_start_dev) {
        // moving window: k_blocks finds the blocks of each run's start on the device, in a table sized for every start;
        // the read set is the whole source (every RIR row, all of x, idx, w)
        std::vector<Block> full;
        int n = 0;
        if (!s.aligned || hb) {
            full.resize((size_t)s.nblk_max);
            n = std::min(plan_blocks(s.aligned, hb, it.P, it.N, s.nb, 0, s.nblk_max, full.data()), s.nblk_max);
        }
        s.nblk_max = window_table_cap(full.empty() ? nullptr : full.data(), n, it.N, it.win_len, s.K, it.P, s.nblk_max);
        s.xa = 0; s.xb = it.N; s.ia = 0; s.ib = it.N;
        window_rows(it.P, it.C, s.K, 0, it.mode == SS_STATIC ? 0 : it.P - 1, s.row0, s.rows);
        s.pa = 0; s.pb = it.P - 1;
        return;
    }
    s.tab_host = !s.aligned || hb != nullptr;
    int pa = 0, pb = it.P - 1;                           // all positions unless the trajectory is visible here
    if (s.tab_host) {
        // (a bounds table outside the contract - ascending from 0 to N - may plan more blocks than the table holds)
        std::vector<Block> full((size_t)s.nblk_max);
        const int n = std::min(plan_blocks(s.aligned, hb, it.P, it.N, s.nb, 0, s.nblk_max, full.data()), s.nblk_max);
        const WinSpan w = window_blocks(full.data(), n, ws, we, s.K);
        if (w.k0 < w.k1) {
            s.g0 = w.g0; s.g1 = w.g1; s.k0 = w.k0; s.k1 = w.k1;
            s.nblk_max = w.g1 - w.g0;
            s.xa = std::max(0, full[w.g0].start - kB); s.xb = std::min(it.N, full[w.g1 - 1].start + kB);
            s.ia = full[w.k0].start; s.ib = full[w.k1 - 1].start + full[w.k1 - 1].len;
            if (s.aligned) { pa = full[w.k0].p_lo; pb = full[w.k1 - 1].p_hi; }
            else if (hb) { pa = seg_of(hb, it.P - 1, s.ia); pb = seg_of(hb, it.P - 1, s.ib - 1) + 1; }
        } else {
            // no block meets the window: only a bounds_host outside the contract (ascending from 0 to N) gets here,
            // which the render paths refuse before they plan; size it as if the blocks were found on the device
            s.tab_host = 0;
        }
    }
    if (!s.tab_host) {
        // k_blocks finds the blocks on the device, in a table that holds them wherever the window lies
        s.nblk_max = window_table_cap(nullptr, 0, it.N, it.win_len, s.K, it.P, s.nblk_max);
        s.xa = 0; s.xb = it.N; s.ia = 0; s.ib = it.N;
    }
    if (it.mode == SS_STATIC) { pa = 0; pb = 0; }
    window_rows(it.P, it.C, s.K, pa, pb, s.row0, s.rows);
    if (it.flags & SS_RIR_NORMALIZE) { s.pa = 0; s.pb = it.P - 1; }         // the global abs-max reads every tap
    else { s.pa = s.row0 / (it.C * s.K); s.pb = (s.row0 + s.rows - 1) / (it.C * s.K); }
}
static Shape shape_of(const ss_source& it) {
    Shape s;
    memset(&s, 0, sizeof(s));
    s.K = (it.L + kB - 1) / kB; s.nb = (it.N + kB - 1) / kB;
    s.aligned = choose_aligned(it, s.K, s.nb) ? 1 : 0;
    s.nblk_max = table_cap(s.aligned, s.nb, it.P);
    s.per = (it.mode == SS_STATIC ? (it.C + 1) / 2 : it.C) * direct_sets(it);
    s.p_max = it.P;
    if (it.win_len > 0) window_shape(it, s);
    s.max_items = s.nblk_max * s.per;
    return s;
}
// A pooled slot: a moving window (tables built by k_blocks, the whole candidate read) under the pool's blocking, sized
// once for the largest table (each candidate with its own K), position count and item count any candidate needs.  The
// table sizes are worked out once per pool and window length.  K is the pool's largest: it picks the kernel variant.
// A slot with a trajectory (traj) is sized for any bounds its runs may take (traj_table_cap).
static Shape shape_pooled(const ss_source& it, bool traj = false) {
    ss_pool* pl = const_cast<ss_pool*>(it.pool);
    Shape s;
    memset(&s, 0, sizeof(s));
    s.K = pl->K; s.aligned = pl->aligned; s.win = 1; s.pooled = 1; s.p_max = pl->p_max; s.traj = traj ? 1 : 0;
    s.per = (it.mode == SS_STATIC ? (it.C + 1) / 2 : it.C) * direct_sets(it);
    s.nblk_max = -1;
    std::vector<std::pair<int, int>>& caps = traj ? pl->traj_caps : pl->caps;
    for (const auto& q : caps) if (q.first == it.win_len) s.nblk_max = q.second;
    if (s.nblk_max < 0 && traj) {
        std::vector<int> N(pl->n), P(pl->n);
        int cap_max = 0;
        for (int i = 0; i < pl->n; ++i) {
            N[i] = pl->host[i].N; P[i] = pl->host[i].P;
            cap_max = std::max(cap_max, table_cap(pl->aligned, (N[i] + kB - 1) / kB, P[i]));
        }
        std::vector<Block> full((size_t)cap_max);
        s.nblk_max = traj_table_cap(pl->aligned, N.data(), P.data(), pl->parts_host.data(), pl->n, it.win_len, pl->K,
                                    full.data());
        caps.push_back({it.win_len, s.nblk_max});
    }
    if (s.nblk_max < 0) {
        std::vector<const int*> bounds;
        std::vector<int> N(pl->n), P(pl->n);
        int cap_max = 0;
        for (int i = 0; i < pl->n; ++i) {
            N[i] = pl->host[i].N; P[i] = pl->host[i].P;
            cap_max = std::max(cap_max, table_cap(pl->aligned, (N[i] + kB - 1) / kB, P[i]));
            if (pl->mode == SS_MOVING_BOUNDS) bounds.push_back(pl->bounds_host.data() + pl->bounds_off[i]);
        }
        std::vector<Block> full((size_t)cap_max);
        s.nblk_max = pool_table_cap(pl->aligned, bounds.empty() ? nullptr : bounds.data(), N.data(), P.data(),
                                    pl->parts_host.data(), pl->n, it.win_len, pl->K, full.data());
        pl->caps.push_back({it.win_len, s.nblk_max});
    }
    s.max_items = s.nblk_max * s.per;
    return s;
}
// RIR rows transformed per set
static size_t rir_rows(const ss_source& it, const Shape& sh) { return sh.win ? (size_t)sh.rows : (size_t)it.P * it.C * sh.K; }
static size_t spectra_bytes(const ss_source& it, const Shape& sh) {
    return (rir_rows(it, sh) * scratch_sets(it) + sh.nblk_max) * kSpec * sizeof(float2) +
           (size_t)sh.max_items * sizeof(RItem) +
           align_up(sizeof(Block) * (size_t)sh.nblk_max, 256) + align_up(sizeof(double) * (size_t)sh.p_max, 256) + 256 +
           ((it.flags & SS_RIR_NORMALIZE) ? 512 : 0) + cut_bytes(it);
}

// Host-side twin of k_blocks for one source whose trajectory bounds are visible on the host.
// Returns the number of blocks in use (windowed source: the full table's blocks [g0, g1)).
static int build_blocks_host(const ss_source& it, const Shape& sh, const int32_t* hb, Block* blocks, double* rstep) {
    const int g0 = sh.win ? sh.g0 : 0, g1 = sh.win ? sh.g1 : sh.nblk_max;
    const int nblk = std::min(plan_blocks(sh.aligned, hb, it.P, it.N, sh.nb, g0, g1, blocks), g1) - g0;
    clear_blocks(blocks, nblk, sh.nblk_max, 0, 1);
    if (it.mode == SS_MOVING_BOUNDS && hb) fill_rstep(hb, it.P, rstep, 0, 1);
    return nblk;
}

// Test hook (pure host, no CUDA call): the blocking plan the library would use for `item` - the choice between
// waypoint-aligned and 4096-grid blocking and the block table of the host-built path.  blocks_out receives
// (start, len, p_lo, p_hi) per block in use; returns their number or a negative ss_status.  Windowed item: the
// entries of the full table that meet the window.
extern "C" int ss_debug_plan(const ss_source* item, int32_t* blocks_out, int32_t max_blocks, int32_t* aligned_out) {
    if (!item || !blocks_out || max_blocks < 0) return SS_ERR_INVALID;
    if (item->N <= 0 || item->C <= 0 || item->L <= 0 || item->P <= 0) return SS_ERR_INVALID;
    if (item->mode == SS_MOVING_BOUNDS && (!item->bounds_host || item->P < 2)) return SS_ERR_INVALID;
    if (item->mode == SS_MOVING_BOUNDS && !bounds_ok(item->bounds_host, item->P, item->N)) return SS_ERR_INVALID;
    if (item->win_len < 0 || item->win_start < 0 || (item->win_len == 0 && item->win_start != 0) ||
        (int64_t)item->win_start + item->win_len > (int64_t)item->N || item->win_start_dev || item->pool ||
        item->pick_dev)
        return SS_ERR_INVALID;
    const Shape sh = shape_of(*item);
    const int first = sh.win ? sh.k0 - sh.g0 : 0;
    const int nout = sh.win ? sh.k1 - sh.k0 : -1;
    if ((sh.win ? nout : sh.nblk_max) > max_blocks) return SS_ERR_NOMEM;
    std::vector<Block> blocks((size_t)sh.nblk_max);
    std::vector<double> rstep((size_t)item->P);
    const int n_tab = build_blocks_host(*item, sh, item->bounds_host, blocks.data(), rstep.data());
    const int nblk = sh.win ? nout : n_tab;
    for (int i = 0; i < nblk; ++i) {
        const Block& b = blocks[first + i];
        blocks_out[4 * i] = b.start; blocks_out[4 * i + 1] = b.len;
        blocks_out[4 * i + 2] = b.p_lo; blocks_out[4 * i + 3] = b.p_hi;
    }
    if (aligned_out) *aligned_out = sh.aligned;
    return nblk;
}

// ---- one chunk of sources = one (k_blocks,) k_prepare, k_render launch group
// Everything the launches need besides the descriptor block in device memory.
struct ChunkLaunch {
    int n = 0, ps = 0, grid_r = 0, n_known = -1;
    int grid_direct = 0;                  // k_rir_direct CTAs per source (8 rows each), 0: no direct target in the chunk
    bool host_tables = true, any_long = false, all_aligned = true, any_norm = false;
    bool any_gain = false;                // a pooled slot of a pool with gains or with pair gains: k_render_fast<true>
    const Source* ds = nullptr; const int* dps = nullptr; RItem* d_items = nullptr; int* d_total = nullptr;
    PrepParams pp;
};
// A chunk is items[first, last) with their shapes at shapes[first, last), worked out once per call (shape_of).
static size_t chunk_scratch_bytes(const ss_source* items, const Shape* shapes, int first, int last) {
    size_t need = 256;
    for (int i = first; i < last; ++i) need += spectra_bytes(items[i], shapes[i]);
    return need;
}
// Block tables on the host when every trajectory is host-visible, every window fixed and no candidate picked on the
// device (always true on the host path)
static bool chunk_host_tables(const ss_source* items, int first, int last) {
    for (int i = first; i < last; ++i)
        if ((items[i].mode == SS_MOVING_BOUNDS && !items[i].bounds_host) || items[i].win_start_dev || items[i].pool)
            return false;
    return true;
}
// counts of a source (Source::counts): [0, 1] and, windowed, [2, 15] - which the host fills even when k_blocks builds the
// block table, so that they always travel in the descriptor block - and for a pooled slot [16..17] (pool_parts),
// [18..19] (stage_view), [20..24] (dry_table, dry_pick_ptr, dry_size) and [26..27] (pair_table), 112 bytes; with a
// trajectory also [25] and [28..31] (has_traj, traj_path, traj_bounds), 128 bytes
static size_t counts_bytes(const Shape& sh) { return sh.traj ? 128 : sh.pooled ? 112 : sh.win ? 64 : 16; }
static const float kUnitGain = 1.0f;      // counts[11] of every windowed source until a pooled slot picks (stem_gain)
// descriptor block: Source[n] | prefix_prepare[n+1] | total | per source: blocks, rstep, counts (host-built tables) or
// counts (windowed source, device-built tables)
static size_t chunk_desc_bytes(const ss_source* items, const Shape* shapes, int first, int last) {
    const int n = last - first;
    size_t bytes = align_up(sizeof(Source) * n, 16) + align_up(sizeof(int) * (n + 1), 16) + 16;
    const bool host_tables = chunk_host_tables(items, first, last);
    for (int i = first; i < last; ++i) {
        const Shape& sh = shapes[i];
        if (host_tables)
            bytes += align_up(sizeof(Block) * (size_t)sh.nblk_max, 16) + align_up(sizeof(double) * (size_t)sh.p_max, 16) +
                     counts_bytes(sh);
        else if (sh.win)
            bytes += counts_bytes(sh);
    }
    return bytes;
}
// What a plan knows of one of its items besides the ss_source: its dry pick, pair gains, dry stream, background
// stream, loudness target and layout draw (validate_dry_picks, validate_streams, validate_bgs, validate_lufs,
// validate_layouts) and, once plan_build has laid out the plan's descriptors,
// the device addresses of its staging area's view (a staged slot), of its DryStream (a stream slot) and of its BgStream
// (a bed slot)
struct PlanSlot {
    const ss_dry_pick* dry = nullptr;
    const float* pair = nullptr;       // the device table of its pair gains, or null
    const ss_dry_stream* strm = nullptr;
    const ss_bg_stream* bg = nullptr;
    const ss_stream_lufs* lufs = nullptr;   // a loudness slot's target (validate_lufs), or null
    const ss_layout_draw* layout = nullptr; // a drawn slot's layout draw (validate_layouts), or null
    const ss_layout_group* group = nullptr; // a drawn stream slot's speaker groups (validate_layouts), or null
    const ss_trajectory* traj = nullptr;    // its trajectory (validate_trajectories), or null
    StageView* view = nullptr;
    const DryStream* ws = nullptr;
    const BgStream* wb = nullptr;
    const ss_dry_pool* clips() const { return strm ? strm->pool : bg ? bg->pool : nullptr; }   // a layout's dry pool
};
// Fill the descriptor block of items[first, last) at `hbase` (host memory) for its device address `dbase`, carve the
// chunk's spectra / tables / work items out of `scratch` (device), and note the launch parameters in `L`.  A plan's
// chunk passes `slots`: slots[first + i] is the record of items[first + i].
static void chunk_describe(const ss_source* items, const Shape* shapes, int first, int last, char* hbase, char* dbase,
                           char* scratch, int sm_count, ChunkLaunch* L, const PlanSlot* const* slots = nullptr) {
    const int n = last - first;
    const bool host_tables = chunk_host_tables(items, first, last);
    const size_t off_ps = align_up(sizeof(Source) * n, 16);
    const size_t off_tot = off_ps + align_up(sizeof(int) * (n + 1), 16);
    Source* hs = (Source*)hbase;
    int* hps = (int*)(hbase + off_ps);
    int ps = 0, pr = 0, total_items = 0;
    size_t tab_off = off_tot + 16;
    bool any_long = false, all_aligned = true, any_norm = false, any_pooled = false;
    int grid_direct = 0;
    L->any_gain = false;
    for (int i = 0; i < n; ++i) {
        const ss_source& it = items[first + i];
        const Shape& sh = shapes[first + i];
        const PlanSlot* const rec = slots ? slots[first + i] : nullptr;
        Source s;
        memset(&s, 0, sizeof(s));
        s.x = it.x; s.rir = it.rir; s.out = it.out;
        s.bounds = it.mode == SS_MOVING_BOUNDS ? it.bounds : nullptr;
        s.idx = it.mode == SS_MOVING_INDEXED ? it.idx : nullptr;
        s.w = it.mode == SS_MOVING_INDEXED ? it.w : nullptr;
        s.N = it.N; s.P = it.P; s.C = it.C; s.L = it.L;
        s.K = sh.K; s.nb = sh.nb; s.mode = it.mode; s.aligned = sh.aligned; s.nblk_max = sh.nblk_max;
        if (it.flags & SS_DIRECT_TARGET) { s.out_direct = it.out_direct; s.direct_taps = it.direct_taps; }
        if (it.pool) {
            // candidate 0 until k_blocks writes the pick of each run over it (the kernel variant below stays the Shape's:
            // the pool's largest K)
            s.K = it.pool->parts_host[0];
            pick_candidate(s, it.pool->host[0]);
            any_pooled = true;
            L->any_gain = L->any_gain || it.pool->gains || (rec && rec->pair);
        } else if (it.rir_bank) {
            // spectra (and cuts) from the bank: no RIR rows, no cut table, no k_rir_absmax / k_rir_direct work
            set_banked(s, it.rir_bank->spec, (it.flags & SS_DIRECT_TARGET) ? it.rir_bank->cut : nullptr, sh.win != 0);
        } else {
            s.hspec = (float2*)scratch; scratch += rir_rows(it, sh) * direct_sets(it) * kSpec * sizeof(float2);
            if (sh.win) { s.h_row0 = sh.row0; s.h_rows = sh.rows; }
        }
        s.xspec = (float2*)scratch; scratch += (size_t)s.nblk_max * kSpec * sizeof(float2);
        if (it.flags & SS_RIR_NORMALIZE) { s.norm_part = (const float*)scratch; scratch += 512; any_norm = true; }
        if ((it.flags & SS_DIRECT_TARGET) && !banked(it)) {
            s.cut = (int*)scratch; scratch += cut_bytes(it);
            grid_direct = std::max(grid_direct, (s.P * s.C + 7) / 8);
        }
        if (host_tables) {
            // tables live in the descriptor block itself: filled here, copied with it
            Block* hb_blocks = (Block*)(hbase + tab_off);
            s.blocks = (Block*)(dbase + tab_off); tab_off += align_up(sizeof(Block) * (size_t)s.nblk_max, 16);
            double* hb_rstep = (double*)(hbase + tab_off);
            s.rstep = (double*)(dbase + tab_off); tab_off += align_up(sizeof(double) * (size_t)sh.p_max, 16);
            int* hb_counts = (int*)(hbase + tab_off);
            s.counts = (int*)(dbase + tab_off); tab_off += counts_bytes(sh);
            memset(hb_counts, 0, counts_bytes(sh));
            const int nblk = build_blocks_host(it, sh, it.bounds_host, hb_blocks, hb_rstep);
            hb_counts[0] = nblk; hb_counts[1] = total_items;
            if (sh.win) {
                hb_counts[2] = sh.k0 - sh.g0; hb_counts[3] = sh.k1 - sh.k0;
                hb_counts[4] = it.win_start; hb_counts[5] = it.win_len;
                memcpy(hb_counts + 11, &kUnitGain, sizeof(kUnitGain));                  // stem_gain
            }
            total_items += (sh.win ? sh.k1 - sh.k0 : nblk) * sh.per;
        } else {
            s.blocks = (Block*)scratch; scratch += align_up(sizeof(Block) * (size_t)s.nblk_max, 256);
            s.rstep = (double*)scratch; scratch += align_up(sizeof(double) * (size_t)sh.p_max, 256);
            if (sh.win) {                               // k_blocks reads the window from the counts and fills [0, 3]
                int* hb_counts = (int*)(hbase + tab_off);
                s.counts = (int*)(dbase + tab_off); tab_off += counts_bytes(sh);
                memset(hb_counts, 0, counts_bytes(sh));
                hb_counts[4] = it.win_start; hb_counts[5] = it.win_len;
                memcpy(hb_counts + 6, &it.win_start_dev, sizeof(it.win_start_dev));      // win_start_ptr
                memcpy(hb_counts + 11, &kUnitGain, sizeof(kUnitGain));                  // stem_gain until k_blocks picks
                if (it.pool) {                              // pool_table, pool_size, pick_ptr, pool_gains, pool_parts
                    memcpy(hb_counts + 8, &it.pool->table, sizeof(it.pool->table));
                    hb_counts[10] = it.pool->n;
                    memcpy(hb_counts + 12, &it.pick_dev, sizeof(it.pick_dev));
                    memcpy(hb_counts + 14, &it.pool->gains, sizeof(it.pool->gains));
                    memcpy(hb_counts + 16, &it.pool->parts, sizeof(it.pool->parts));
                    if (rec) memcpy(hb_counts + 18, &rec->view, sizeof(rec->view));            // stage_view
                    // dry_table, dry_pick_ptr, dry_size, pair_table of the dry picks k_blocks makes (pick_pooled): a
                    // staged slot's is k_stage's, and its counts hold none (take_view)
                    if (rec && rec->dry && !rec->view) {
                        const ss_dry_pick& d = *rec->dry;
                        memcpy(hb_counts + 20, &d.pool->ptrs, sizeof(d.pool->ptrs));
                        memcpy(hb_counts + 22, &d.pick_dev, sizeof(d.pick_dev));
                        hb_counts[24] = d.pool->n;
                        memcpy(hb_counts + 26, &rec->pair, sizeof(rec->pair));
                    }
                    if (rec && rec->traj) {                     // has_traj, traj_path, traj_bounds
                        hb_counts[25] = 1;
                        memcpy(hb_counts + 28, &rec->traj->path_dev, sizeof(rec->traj->path_dev));
                        memcpy(hb_counts + 30, &rec->traj->bounds_dev, sizeof(rec->traj->bounds_dev));
                    }
                }
            } else {
                s.counts = (int*)scratch;
            }
            scratch += 256;
        }
        hs[i] = s;
        hps[i] = ps;
        ps += spectra_pairs_h(s) + spectra_pairs_x(s) + range_ctas(s);
        pr += sh.max_items;
        any_long = any_long || sh.K > 1;
        all_aligned = all_aligned && one_transform_per_item(sh.aligned, it.mode, sh.K);
    }
    hps[n] = ps;
    // work-item table of the whole chunk (dense) + its length
    L->d_items = (RItem*)scratch; scratch += (size_t)pr * sizeof(RItem);
    L->d_total = host_tables ? (int*)(dbase + off_tot) : (int*)scratch;
    if (host_tables) { *(int*)(hbase + off_tot) = total_items; pr = total_items; }
    L->n = n; L->ps = ps; L->host_tables = host_tables; L->any_long = any_long; L->all_aligned = all_aligned;
    L->any_norm = any_norm;
    L->grid_direct = grid_direct;
    L->n_known = host_tables ? total_items : -1;
    L->grid_r = pr < sm_count * SS_RENDER_MINB ? pr : sm_count * SS_RENDER_MINB;
    L->ds = (const Source*)dbase;
    L->dps = (const int*)(dbase + off_ps);
    // a pooled slot's Source is written by k_blocks at every run: k_prepare reads the table from global memory
    L->pp.n_inline = n <= kPrepInline && !any_pooled ? n : 0;
    if (L->pp.n_inline) {
        memcpy(L->pp.prefix, hps, sizeof(int) * (size_t)(n + 1));
        memcpy(L->pp.srcs, hs, sizeof(Source) * (size_t)n);
    }
}
// The kernel launches of one described chunk (its descriptor block is, or will be by stream order, in device memory).
// `timed`: events around its prepare and render launches, for ss_get_profile.
static int chunk_enqueue(ss_ctx* c, const ChunkLaunch& L, cudaStream_t stream, bool timed) {
    ss_ctx::Prof pf = {};
    if (timed) {
        CK(cudaEventCreate(&pf.e0)); CK(cudaEventCreate(&pf.e1)); CK(cudaEventCreate(&pf.e2));
        pf.chunk = c->prof_chunk++;
        c->prof.push_back(pf);
        CK(cudaEventRecord(pf.e0, stream));
    }
    if (!L.host_tables) {
        k_blocks<<<1, 256, 0, stream>>>(const_cast<Source*>(L.ds), L.n, L.d_total, L.d_items);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    if (L.any_norm) {
        k_rir_absmax<<<L.n * kNormParts, 256, 0, stream>>>(L.ds);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    if (L.grid_direct > 0) {
        k_rir_direct<<<L.n * L.grid_direct, 256, 0, stream>>>(L.ds, L.grid_direct);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    if (L.ps > 0) {
        if (L.pp.n_inline) k_prepare<true><<<L.ps, kThreads, kPadF * (int)sizeof(float2), stream>>>(L.ds, L.dps, L.n, L.d_items, L.pp);
        else k_prepare<false><<<L.ps, kThreads, kPadF * (int)sizeof(float2), stream>>>(L.ds, L.dps, L.n, L.d_items, L.pp);
        CK(cudaGetLastError());
    }
    if (timed) CK(cudaEventRecord(pf.e1, stream));
    if (L.grid_r > 0) {
        if (L.any_long) k_render<true, false><<<L.grid_r, kThreads, kRenderSmem, stream>>>(L.d_items, L.d_total, L.n_known);
        else if (L.all_aligned && !c->no_fast) {
            if (L.any_gain) k_render_fast<true><<<L.grid_r, kThreads, kRenderSmem, stream>>>(L.d_items, L.d_total, L.n_known);
            else k_render_fast<false><<<L.grid_r, kThreads, kRenderSmem, stream>>>(L.d_items, L.d_total, L.n_known);
        }
        else k_render<false, false><<<L.grid_r, kThreads, kRenderSmem, stream>>>(L.d_items, L.d_total, L.n_known);
        CK(cudaGetLastError());
    }
    if (timed) CK(cudaEventRecord(pf.e2, stream));
    c->launches += (L.ps > 0 ? 1 : 0) + (L.grid_r > 0 ? 1 : 0);      // (both, for every chunk of a render)
    return SS_OK;
}

// ----------------------------------------------------------------------------- RIR spectrum banks
// A bank is built by the render pipeline itself: one chunk whose only source has the bank's RIRs and no blocks
// (nblk_max = 0), so that k_rir_absmax (SS_RIR_NORMALIZE), k_rir_direct (SS_DIRECT_TARGET) and k_prepare's RIR CTAs run
// exactly as for a whole source of a render - rows paired (2r, 2r + 1) per set - and write into the bank instead of
// chunk scratch.  Its spectra therefore have the bits a render would transform itself.
static int bank_args(const ss_ctx* c, const float* rir, int P, int C, int L, int flags, int direct_taps, ss_bank** out) {
    if (!c || !rir || !out || P < 1 || C < 1 || L < 1) return SS_ERR_INVALID;
    if (flags & ~(SS_RIR_NORMALIZE | SS_DIRECT_TARGET | SS_BANK_HOST | SS_BANK_TAPS)) return SS_ERR_INVALID;
    if ((flags & SS_BANK_TAPS) && !(flags & SS_BANK_HOST)) return SS_ERR_INVALID;     // tap rows: host banks only
    if ((flags & SS_DIRECT_TARGET) && direct_taps < 1) return SS_ERR_INVALID;
    if ((int64_t)P * C * ((L + kB - 1) / kB) > (int64_t)1 << 28) return SS_ERR_UNSUPPORTED;    // as validate_item
    return SS_OK;
}
// SS_BANK_TAPS: the n = P*C*K * kB stored taps (tap_value) from bank_build's blockless source, after k_rir_absmax
__global__ void __launch_bounds__(256) k_bank_taps(const Source* __restrict__ src, float* __restrict__ taps, long long n) {
    const Source& S = *src;
    const float m = S.norm_part ? rir_absmax(S) : 0.f;
    for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < n; q += (long long)gridDim.x * blockDim.x)
        taps[q] = tap_value(S, (int)(q / kB), (int)(q % kB), m);
}
static int bank_build(ss_ctx* c, ss_bank* b, const float* rir, cudaStream_t stream) {
    const bool direct = (b->flags & SS_DIRECT_TARGET) != 0, norm = (b->flags & SS_RIR_NORMALIZE) != 0;
    const bool taps = (b->flags & SS_BANK_TAPS) != 0;
    const size_t spec_b = b->head_bytes(), cut_b = align_up(b->cut_bytes(), 256);
    const size_t src_b = align_up(sizeof(Source), 256);
    b->bytes = spec_b + cut_b + src_b + (norm ? 512 : 0);
    CK(cudaMalloc((void**)&b->d_mem, b->bytes));
    char* p = b->d_mem;
    b->spec = (float2*)p; p += spec_b;
    if (direct) { b->cut = (int*)p; p += cut_b; }
    Source* d_src = (Source*)p; p += src_b;
    Source s;
    memset(&s, 0, sizeof(s));
    s.rir = rir; s.N = 1; s.P = b->P; s.C = b->C; s.L = b->L; s.K = b->K; s.nb = 1;
    s.mode = b->P == 1 ? MODE_STATIC : MODE_MOVING_BOUNDS;
    s.nblk_max = 0;                                      // no blocks: no dry windows, no range CTAs, no items
    s.hspec = b->spec;
    if (norm) s.norm_part = (const float*)p;
    if (direct) { s.cut = b->cut; s.direct_taps = b->direct_taps; }
    static thread_local ChunkLaunch L;                  // kernel parameters, as in launch_chunk
    L = ChunkLaunch();
    L.n = 1; L.ps = taps ? 0 : spectra_pairs_h(s); L.grid_r = 0; L.n_known = 0;   // (tap rows: no transform)
    L.any_norm = norm; L.grid_direct = direct ? (s.P * s.C + 7) / 8 : 0;
    L.ds = d_src;
    L.pp.n_inline = 1; L.pp.prefix[0] = 0; L.pp.prefix[1] = L.ps; L.pp.srcs[0] = s;
    CK(cudaEventCreateWithFlags(&b->ready, cudaEventDisableTiming));
    CK(cudaMemcpyAsync(d_src, &s, sizeof(s), cudaMemcpyHostToDevice, stream));  // k_rir_absmax / k_rir_direct read it
    { int st = chunk_enqueue(c, L, stream, false); if (st) return st; }
    if (taps) {
        const long long n = (long long)b->P * b->C * b->K * kB;
        k_bank_taps<<<(unsigned)std::min(n / 256, (long long)c->sm_count * 8), 256, 0, stream>>>(d_src, (float*)b->spec, n);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    CK(cudaEventRecord(b->ready, stream));
    return SS_OK;
}
// SS_BANK_HOST: the built spectra (SS_BANK_TAPS: tap rows) and cut table into pinned, mapped host memory, then the
// device buffer freed.  Returns when the bank is in host memory.
static int bank_to_host(ss_bank* b, cudaStream_t stream) {
    const size_t spec_b = b->head_bytes(), cut_b = b->cut_bytes();
    CK(cudaHostAlloc((void**)&b->h_mem, spec_b + cut_b, cudaHostAllocMapped | cudaHostAllocPortable));
    b->host_bytes = spec_b + cut_b;
    CK(cudaMemcpyAsync(b->h_mem, b->spec, spec_b, cudaMemcpyDeviceToHost, stream));
    if (cut_b) CK(cudaMemcpyAsync(b->h_mem + spec_b, b->cut, cut_b, cudaMemcpyDeviceToHost, stream));
    CK(cudaStreamSynchronize(stream));
    CK(cudaFree(b->d_mem));
    b->d_mem = nullptr; b->bytes = 0;
    char* dev = nullptr;
    CK(cudaHostGetDevicePointer((void**)&dev, b->h_mem, 0));
    b->spec = (float2*)dev;
    b->cut = cut_b ? (int*)(dev + spec_b) : nullptr;
    return SS_OK;
}

// Waits for the whole device: a render that used the bank may run on any stream of the caller (cudaFree would wait for
// the device anyway).
extern "C" void ss_bank_destroy(ss_bank* b) {
    if (!b) return;
    cudaSetDevice(b->c->device);
    cudaDeviceSynchronize();
    if (b->d_mem) cudaFree(b->d_mem);
    if (b->h_mem) cudaFreeHost(b->h_mem);
    if (b->ready) cudaEventDestroy(b->ready);
    delete b;
}
extern "C" int64_t ss_bank_bytes(const ss_bank* b) { return b ? (int64_t)b->bytes : 0; }
extern "C" int64_t ss_bank_host_bytes(const ss_bank* b) { return b ? (int64_t)b->host_bytes : 0; }
extern "C" int32_t ss_bank_flags(const ss_bank* b) { return b ? b->flags : 0; }

extern "C" int ss_bank_create_dev(ss_ctx* c, const float* rir, int32_t P, int32_t C, int32_t L, int32_t flags,
                                  int32_t direct_taps, void* stream, ss_bank** out) {
    { int st = bank_args(c, rir, P, C, L, flags, direct_taps, out); if (st) return st; }
    *out = nullptr;
    CK(cudaSetDevice(c->device));
    ss_bank* b = new (std::nothrow) ss_bank();
    if (!b) return SS_ERR_NOMEM;
    b->c = c; b->P = P; b->C = C; b->L = L; b->K = (L + kB - 1) / kB; b->flags = flags;
    b->direct_taps = (flags & SS_DIRECT_TARGET) ? direct_taps : 0;
    int st = bank_build(c, b, rir, (cudaStream_t)stream);
    if (st == SS_OK && (flags & SS_BANK_HOST)) st = bank_to_host(b, (cudaStream_t)stream);
    if (st != SS_OK) { ss_bank_destroy(b); return st; }
    *out = b;
    return SS_OK;
}

extern "C" int ss_bank_create_host(ss_ctx* c, const float* rir, int32_t P, int32_t C, int32_t L, int32_t flags,
                                   int32_t direct_taps, ss_bank** out) {
    { int st = bank_args(c, rir, P, C, L, flags, direct_taps, out); if (st) return st; }
    *out = nullptr;
    CK(cudaSetDevice(c->device));
    // the RIRs pass through the host path's first input slot, idle between calls (ss_render_host_ex returns after its
    // streams): no allocation per bank once the slot is large enough
    const size_t nb = sizeof(float) * (size_t)P * C * L;
    ss_ctx::Slot& sl = c->slot[0];
    { int st = ensure(&sl.d_in, &sl.in_cap, nb); if (st) return st; }
    const float* d_rir = (const float*)sl.d_in;
    int st = SS_OK;
    cudaError_t e = cudaMemcpyAsync(sl.d_in, rir, nb, cudaMemcpyHostToDevice, c->s_in);
    if (e != cudaSuccess) { g_last_cuda = (int)e; st = SS_ERR_CUDA; }
    if (st == SS_OK) st = ss_bank_create_dev(c, d_rir, P, C, L, flags, direct_taps, (void*)c->s_in, out);
    e = cudaStreamSynchronize(c->s_in);                 // the bank is complete; the slot is free again
    if (st == SS_OK && e != cudaSuccess) { g_last_cuda = (int)e; st = SS_ERR_CUDA; }
    if (st != SS_OK && *out) { ss_bank_destroy(*out); *out = nullptr; }
    return st;
}

// ----------------------------------------------------------------------------- source pools
// A candidate of a pool (include/sonicsim_b200.h): a banked source of this context, moving over host-visible bounds or
// static, with none of a slot's fields.
static int validate_candidate(const ss_ctx* c, const ss_source& it) {
    if (!it.x || it.rir || !it.rir_bank || it.rir_bank->c != c || it.idx || it.w) return SS_ERR_INVALID;
    if (it.out || it.out_direct || it.flags || it.direct_taps || it.win_start || it.win_len || it.win_start_dev ||
        it.pool || it.pick_dev)
        return SS_ERR_INVALID;
    if (it.N <= 0 || it.C <= 0 || it.L <= 0 || it.P <= 0) return SS_ERR_INVALID;
    if (it.N > 0x7fffffff - 2 * kF) return SS_ERR_INVALID;                 // as validate_item
    if (it.mode == SS_STATIC) { if (it.P != 1 || it.bounds || it.bounds_host) return SS_ERR_INVALID; }
    else if (it.mode == SS_MOVING_BOUNDS) {
        // (a host pool uploads bounds_host itself: its candidates need no device bounds)
        if (it.P < 2 || (!it.bounds && !it.rir_bank->h_mem) || !it.bounds_host || !bounds_ok(it.bounds_host, it.P, it.N))
            return SS_ERR_INVALID;
    } else return SS_ERR_INVALID;
    return bank_fits(it);
}

// the level tables (pinned, mapped host memory in a host pool) and their pointer array
static void free_levels(ss_pool* pl) {
    if (pl->levels) { if (pl->host_res) cudaFreeHost(pl->h_levels); else cudaFree(pl->levels); }
    if (pl->level_ptr) cudaFree(pl->level_ptr);
    pl->levels = nullptr; pl->h_levels = nullptr; pl->level_ptr = nullptr;
}
extern "C" void ss_pool_destroy(ss_pool* pl) {
    if (!pl) return;
    cudaSetDevice(pl->c->device);
    cudaDeviceSynchronize();                            // (a plan that used it may run on any stream)
    if (pl->table) cudaFree(pl->table);
    if (pl->parts) cudaFree(pl->parts);
    free_levels(pl);
    if (pl->gains) cudaFree(pl->gains);
    if (pl->ready) cudaEventDestroy(pl->ready);
    if (pl->h_x) cudaFreeHost(pl->h_x);
    if (pl->d_aux) cudaFree(pl->d_aux);
    delete pl;
}
static size_t level_bytes(const ss_pool* pl) { return sizeof(double) * (size_t)pl->level_off[pl->n]; }
extern "C" int64_t ss_pool_bytes(const ss_pool* pl) {
    if (!pl) return 0;
    int64_t b = (int64_t)sizeof(PoolEntry) * pl->n;
    if (pl->parts) b += (int64_t)sizeof(int) * pl->n;
    if (pl->levels) b += (pl->host_res ? 0 : (int64_t)level_bytes(pl)) + (int64_t)sizeof(double*) * pl->n;
    if (pl->gains) b += (int64_t)sizeof(float) * pl->n;
    return b + (int64_t)pl->aux_bytes;
}
extern "C" int64_t ss_pool_host_bytes(const ss_pool* pl) {
    return pl && pl->host_res ? (int64_t)(pl->h_x_bytes + (pl->levels ? level_bytes(pl) : 0)) : 0;
}
extern "C" const double* ss_pool_level_table(const ss_pool* pl, int i) {
    return pl && pl->levels && i >= 0 && i < pl->n ? pl->levels + pl->level_off[i] : nullptr;
}

// Host pool: the candidates' x into the pool's pinned, mapped arena (each at a 64-byte boundary, zero-padded to a multiple
// of 4 samples: k_stage copies whole float4s), bounds_host and the banks' cut tables into one device allocation; the
// entries point at the device addresses of both.
static int pool_host_copies(ss_pool* pl, const ss_source* cand) {
    const int n = pl->n;
    std::vector<size_t> xo(n + 1, 0), ao(n + 1, 0);
    for (int i = 0; i < n; ++i) {
        xo[i + 1] = xo[i] + align_up(sizeof(float) * (size_t)cand[i].N, 64);
        const ss_bank* b = cand[i].rir_bank;
        ao[i + 1] = ao[i] + (pl->mode == SS_MOVING_BOUNDS ? (size_t)cand[i].P : 0) + b->cut_bytes() / sizeof(int);
    }
    pl->h_x_bytes = xo[n];
    CK(cudaHostAlloc((void**)&pl->h_x, pl->h_x_bytes, cudaHostAllocMapped | cudaHostAllocPortable));
    memset(pl->h_x, 0, pl->h_x_bytes);
    char* dx = nullptr;
    CK(cudaHostGetDevicePointer((void**)&dx, pl->h_x, 0));
    std::vector<int> aux(ao[n]);
    for (int i = 0; i < n; ++i) {
        const ss_bank* b = cand[i].rir_bank;
        int* a = aux.data() + ao[i];
        if (pl->mode == SS_MOVING_BOUNDS) { memcpy(a, cand[i].bounds_host, sizeof(int) * (size_t)cand[i].P); a += cand[i].P; }
        if (b->cut) memcpy(a, b->h_mem + b->head_bytes(), b->cut_bytes());
        CK(cudaMemcpy(pl->h_x + xo[i], cand[i].x, sizeof(float) * (size_t)cand[i].N, cudaMemcpyDefault));
    }
    pl->aux_bytes = sizeof(int) * std::max(ao[n], (size_t)1);
    CK(cudaMalloc((void**)&pl->d_aux, pl->aux_bytes));
    if (ao[n]) CK(cudaMemcpy(pl->d_aux, aux.data(), sizeof(int) * ao[n], cudaMemcpyHostToDevice));
    for (int i = 0; i < n; ++i) {
        PoolEntry& e = pl->host[i];
        int* a = pl->d_aux + ao[i];
        e.x = (const float*)(dx + xo[i]);
        if (pl->mode == SS_MOVING_BOUNDS) { e.bounds = a; a += cand[i].P; }
        e.cut = e.cut ? a : nullptr;
    }
    return SS_OK;
}

static int pool_build(ss_pool* pl, const ss_source* cand) {
    ss_ctx* c = pl->c;
    const ss_source& a = cand[0];
    pl->mode = a.mode; pl->C = a.C; pl->L = a.L; pl->K = a.rir_bank->K; pl->aligned = 1;
    pl->n_min = a.N; pl->direct_taps = a.rir_bank->cut ? a.rir_bank->direct_taps : 0;
    pl->host.resize(pl->n);
    pl->parts_host.resize(pl->n);
    if (pl->mode == SS_MOVING_BOUNDS) pl->bounds_off.resize(pl->n);
    std::vector<ss_bank*> banks;
    for (int i = 0; i < pl->n; ++i) {
        const ss_source& it = cand[i];
        const ss_bank* b = it.rir_bank;
        PoolEntry e;
        e.x = it.x; e.bounds = it.mode == SS_MOVING_BOUNDS ? it.bounds : nullptr; e.spec = b->spec; e.cut = b->cut;
        e.N = it.N; e.P = it.P;
        pl->host[i] = e;
        pl->n_min = std::min(pl->n_min, it.N); pl->p_max = std::max(pl->p_max, it.P);
        pl->L = std::max(pl->L, it.L); pl->K = std::max(pl->K, b->K); pl->parts_host[i] = b->K;
        if (pl->direct_taps != (b->cut ? b->direct_taps : 0)) pl->direct_taps = 0;
        // the pool's blocking: aligned only if every candidate would choose it with its own K
        if (!choose_aligned(it, b->K, (it.N + kB - 1) / kB)) pl->aligned = 0;
        if (pl->mode == SS_MOVING_BOUNDS) {
            pl->bounds_off[i] = (int64_t)pl->bounds_host.size();
            pl->bounds_host.insert(pl->bounds_host.end(), it.bounds_host, it.bounds_host + it.P);
        }
        if (std::find(banks.begin(), banks.end(), b) == banks.end()) banks.push_back(const_cast<ss_bank*>(b));
        pl->banks.push_back(b);
    }
    if (pl->host_res) { int st = pool_host_copies(pl, cand); if (st) return st; }
    CK(cudaMalloc((void**)&pl->table, sizeof(PoolEntry) * (size_t)pl->n));
    CK(cudaMemcpy(pl->table, pl->host.data(), sizeof(PoolEntry) * (size_t)pl->n, cudaMemcpyHostToDevice));
    if (std::any_of(pl->parts_host.begin(), pl->parts_host.end(), [&](int k) { return k != pl->K; })) {
        CK(cudaMalloc((void**)&pl->parts, sizeof(int) * (size_t)pl->n));
        CK(cudaMemcpy(pl->parts, pl->parts_host.data(), sizeof(int) * (size_t)pl->n, cudaMemcpyHostToDevice));
    }
    // one event behind every bank's construction: a plan run waits once per pool, not once per candidate bank
    CK(cudaEventCreateWithFlags(&pl->ready, cudaEventDisableTiming));
    cudaStream_t s = nullptr;
    CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
    int st = SS_OK;
    for (ss_bank* b : banks) {
        const cudaError_t e = cudaStreamWaitEvent(s, b->ready, 0);
        if (e != cudaSuccess) { g_last_cuda = (int)e; st = SS_ERR_CUDA; break; }
    }
    if (st == SS_OK) {
        const cudaError_t e = cudaEventRecord(pl->ready, s);
        if (e != cudaSuccess) { g_last_cuda = (int)e; st = SS_ERR_CUDA; }
    }
    cudaStreamDestroy(s);                               // (the recorded work completes on its own)
    return st;
}

extern "C" int ss_pool_create(ss_ctx* c, const ss_source* cand, int n, ss_pool** out) {
    if (!c || !cand || !out || n < 1 || n > (1 << 24)) return SS_ERR_INVALID;
    *out = nullptr;
    for (int i = 0; i < n; ++i) {
        const int st = validate_candidate(c, cand[i]);
        if (st) return st;
        if (cand[i].mode != cand[0].mode || cand[i].C != cand[0].C) return SS_ERR_INVALID;   // any L
        if (!cand[i].rir_bank->h_mem != !cand[0].rir_bank->h_mem) return SS_ERR_INVALID;  // host and device banks
        if ((cand[i].rir_bank->flags ^ cand[0].rir_bank->flags) & SS_BANK_TAPS) return SS_ERR_INVALID;   // two forms
    }
    CK(cudaSetDevice(c->device));
    ss_pool* pl = new (std::nothrow) ss_pool();
    if (!pl) return SS_ERR_NOMEM;
    pl->c = c; pl->n = n; pl->host_res = cand[0].rir_bank->h_mem != nullptr;
    pl->taps = (cand[0].rir_bank->flags & SS_BANK_TAPS) != 0;
    const int st = pool_build(pl, cand);
    if (st != SS_OK) { ss_pool_destroy(pl); return st; }
    *out = pl;
    return SS_OK;
}

// Describe items[first, last) (device pointers) in the next slot of the descriptor ring, copy the block and enqueue
// the launches on `stream`, with scratch buffer `buf`.
static int launch_chunk(ss_ctx* c, const ss_source* items, const Shape* shapes, int first, int last,
                        cudaStream_t stream, int buf) {
    const size_t need = chunk_scratch_bytes(items, shapes, first, last);
    { const int st = ensure(&c->d_scratch[buf], &c->scratch_cap[buf], need); if (st) return st; }
    const size_t bytes = chunk_desc_bytes(items, shapes, first, last);
    int slot; char *hblk, *dblk;
    { int st = ring_acquire(c, bytes, stream, &slot, &hblk, &dblk); if (st) return st; }
    static thread_local ChunkLaunch L;                  // holds 3.2 KB of kernel parameters: not on the stack
    chunk_describe(items, shapes, first, last, hblk, dblk, c->d_scratch[buf], c->sm_count, &L);
    CK(cudaMemcpyAsync(dblk, hblk, bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaEventRecord(c->desc_ev[slot], stream));
    const int st = chunk_enqueue(c, L, stream, c->profiling);
    const int rs = ring_release(c, slot, stream);
    return st ? st : rs;
}

// split [0, n) into chunks whose spectra fit the L2-sized budget
static void make_chunks_bytes(const std::vector<size_t>& sb, int64_t budget, std::vector<int>& cuts) {
    const int n = (int)sb.size();
    // greedy pass: how many chunks does the budget need ...
    size_t total = 0, acc = 0;
    int n_chunks = 1;
    for (int i = 0; i < n; ++i) {
        total += sb[i];
        if (acc > 0 && acc + sb[i] > (size_t)budget) { ++n_chunks; acc = 0; }
        acc += sb[i];
    }
    // ... then cut at equal shares of the total, so that the last chunk is not a runt (7,7,7,7,4 -> 6,6,7,6,7):
    // equal chunks keep the streams of the overlap equally busy.  A chunk never exceeds the budget (measured from
    // the bytes accumulated at its own first item) unless a single item does.
    cuts.clear(); cuts.push_back(0);
    acc = 0;
    size_t chunk_start = 0;                            // bytes in front of the current chunk
    for (int i = 0; i < n; ++i) {
        const size_t target = total * cuts.size() / n_chunks;
        if (i > cuts.back() && (acc + sb[i] / 2 > target || acc - chunk_start + sb[i] > (size_t)budget)) {
            cuts.push_back(i);
            chunk_start = acc;
        }
        acc += sb[i];
    }
    cuts.push_back(n);
}
static void make_chunks(const ss_source* items, const Shape* shapes, int n, int64_t budget, std::vector<int>& cuts) {
    std::vector<size_t> sb(n);
    for (int i = 0; i < n; ++i) sb[i] = spectra_bytes(items[i], shapes[i]);
    make_chunks_bytes(sb, budget, cuts);
}
// Device path: sources are independent, so a batch is regrouped by the kernel variant its chunk would run - one
// transform per item (aligned moving sources and static ones: k_render_fast), long RIRs (k_render<LONG>), everything
// else (k_render<0, 0>) - and each group
// is chunked on its own: one static source no longer sends the moving sources of its chunk through the generic kernel
// (a SonicSet scene is 3 moving + 2 static sources).  `arranged` / `arranged_shapes` receive the regrouped items and
// their shapes, `cuts` the chunk bounds, and `order` (when given) the caller's index of every arranged item.
static void arrange_chunks(const ss_ctx* c, const ss_source* items, const Shape* shapes, int n,
                           std::vector<ss_source>& arranged, std::vector<Shape>& arranged_shapes, std::vector<int>& cuts,
                           std::vector<int>* order = nullptr) {
    arranged.clear(); arranged.reserve(n);
    arranged_shapes.clear(); arranged_shapes.reserve(n);
    cuts.clear(); cuts.push_back(0);
    if (order) order->clear();
    for (int cls = 0; cls < 3; ++cls) {
        const int lo = (int)arranged.size();
        for (int i = 0; i < n; ++i) {
            const Shape& sh = shapes[i];
            const int k = sh.K > 1 ? 1 : (one_transform_per_item(sh.aligned, items[i].mode, sh.K) ? 0 : 2);
            if (k == cls) {
                arranged.push_back(items[i]); arranged_shapes.push_back(sh);
                if (order) order->push_back(i);
            }
        }
        const int cnt = (int)arranged.size() - lo;
        if (cnt == 0) continue;
        std::vector<int> local;
        make_chunks(arranged.data() + lo, arranged_shapes.data() + lo, cnt, c->chunk_bytes, local);
        for (size_t q = 1; q < local.size(); ++q) cuts.push_back(lo + local[q]);
    }
}
// Test hook (pure host): the chunking of items whose scratch needs are `bytes[i]` under `budget`; cuts_out receives
// the first item of every chunk plus n (at most max_cuts values); returns the number of values written or a negative status.
extern "C" int ss_debug_chunks(const int64_t* bytes, int32_t n, int64_t budget, int32_t* cuts_out, int32_t max_cuts) {
    if (!bytes || !cuts_out || n <= 0 || budget <= 0) return SS_ERR_INVALID;
    std::vector<size_t> sb(n);
    for (int i = 0; i < n; ++i) { if (bytes[i] <= 0) return SS_ERR_INVALID; sb[i] = (size_t)bytes[i]; }
    std::vector<int> cuts;
    make_chunks_bytes(sb, budget, cuts);
    if ((int)cuts.size() > max_cuts) return SS_ERR_NOMEM;
    for (size_t i = 0; i < cuts.size(); ++i) cuts_out[i] = cuts[i];
    return (int)cuts.size();
}

// Validate a device-path batch and work out the shape of every source, once per call.  Pooled slots only in plans.
static int shape_dev_items(const ss_ctx* c, const ss_source* items, int n_items, std::vector<Shape>& shapes,
                           bool pools_ok) {
    shapes.resize(n_items);
    for (int i = 0; i < n_items; ++i) {
        if (pools_ok && items[i].pool) {
            const int st = validate_pooled(c, items[i]); if (st) return st;
            shapes[i] = shape_pooled(items[i]);
            continue;
        }
        int st = validate_item_ctx(c, items[i]); if (st) return st;
        if (items[i].mode == SS_MOVING_BOUNDS && items[i].bounds_host &&
            !bounds_ok(items[i].bounds_host, items[i].P, items[i].N))
            return SS_ERR_INVALID;
        shapes[i] = shape_of(items[i]);
    }
    return SS_OK;
}

// Profiling: let the host enqueue a call's launches while the GPU idles, so that no timed interval contains a wait for
// the host; chunk positions restart for the grouping in ss_get_profile.
static int profile_start(ss_ctx* c, cudaStream_t stream) {
    c->prof_chunk = 0;
    k_delay<<<1, 1, 0, stream>>>(300000u);
    CK(cudaGetLastError());
    return SS_OK;
}
// Chunks run one after another on the caller's stream when there is only one, under SS_SINGLE_STREAM, and while
// profiling (serialised kernels give clean per-kernel times).
static bool chunks_serial(const ss_ctx* c, size_t n_chunks) { return n_chunks < 2 || c->single_stream || c->profiling; }
// Enqueue chunks [0, n_chunks) behind `stream` through run(k, stream, scratch buffer): serially on `stream` with buffer
// 0, or chunk k on internal stream and buffer k % kAux, forked from `stream` at ev_fork and joined back into it.  When
// it returns, ev_join[i] marks the last use of buffer i (serially: ev_join[0]).
template <class Run>
static int run_chunks(ss_ctx* c, size_t n_chunks, cudaStream_t stream, cudaEvent_t ev_fork, const cudaEvent_t* ev_join,
                      Run run) {
    if (chunks_serial(c, n_chunks)) {
        for (size_t k = 0; k < n_chunks; ++k) { int st = run(k, stream, 0); if (st) return st; }
        CK(cudaEventRecord(ev_join[0], stream));
        return SS_OK;
    }
    CK(cudaEventRecord(ev_fork, stream));
    for (int i = 0; i < ss_ctx::kAux; ++i) CK(cudaStreamWaitEvent(c->s_aux[i], ev_fork, 0));
    int rc = SS_OK;
    for (size_t k = 0; k < n_chunks && rc == SS_OK; ++k) rc = run(k, c->s_aux[k % ss_ctx::kAux], (int)(k % ss_ctx::kAux));
    for (int i = 0; i < ss_ctx::kAux; ++i) {
        CK(cudaEventRecord(ev_join[i], c->s_aux[i]));
        CK(cudaStreamWaitEvent(stream, ev_join[i], 0));
    }
    return rc;
}

extern "C" int ss_render_dev(ss_ctx* c, const ss_source* items, int n_items, void* stream_) {
    if (!c || (!items && n_items > 0) || n_items < 0) return SS_ERR_INVALID;
    if (n_items == 0) return SS_OK;
    CK(cudaSetDevice(c->device));
    const cudaStream_t stream = (cudaStream_t)stream_;
    std::vector<Shape> shapes;
    { int st = shape_dev_items(c, items, n_items, shapes, false); if (st) return st; }
    { int st = wait_banks(items, n_items, stream); if (st) return st; }   // before the fork: every chunk
    // the scratch buffers' last users, on whatever stream the previous call ran (a no-op wait on the same stream)
    for (int i = 0; i < ss_ctx::kAux; ++i) CK(cudaStreamWaitEvent(stream, c->ev_join[i], 0));
    std::vector<int> cuts;
    std::vector<ss_source> arranged;
    std::vector<Shape> arranged_shapes;
    arrange_chunks(c, items, shapes.data(), n_items, arranged, arranged_shapes, cuts);
    const size_t n_chunks = cuts.size() - 1;
    if (c->profiling) { int st = profile_start(c, stream); if (st) return st; }
    if (!chunks_serial(c, n_chunks)) c->ring_pos = 0;  // forked: descriptor ring slot k % kRing <-> stream k % kAux
    return run_chunks(c, n_chunks, stream, c->ev_fork, c->ev_join, [&](size_t k, cudaStream_t s, int buf) {
        return launch_chunk(c, arranged.data(), arranged_shapes.data(), cuts[k], cuts[k + 1], s, buf);
    });
}

// ----------------------------------------------------------------------------- whole stems of a pool's candidates
// ss_pool_loudness, ss_pool_levels and ss_pair_gains_create read whole reverberant stems as ss_render_dev renders them
// (the candidate as a whole banked source, bounds_host included).  A stem is a candidate rendered with one dry signal:
// its own x, or (ss_pair_gains_create) the first N samples of a dry pool's signal.  The stems are rendered in groups of
// consecutive stems whose outputs fit kLevelStemBytes (a larger stem is a group of its own) into one transient buffer.
constexpr size_t kLevelStemBytes = 256ull << 20;

struct Stem { int cand, sig; };           // candidate `cand` with signal `sig` of the dry pool, or sig < 0: its own x
struct StemSet {
    const ss_pool* pl = nullptr;
    const ss_dry_pool* dry = nullptr;     // the pool the signals come from, or null: every stem takes its own x
    std::vector<Stem> stems;
    int N(size_t k) const { return pl->host[stems[k].cand].N; }
    // (null for a 16-bit signal, which is only read through its float32 expansion: render_copied_stems)
    const float* x(size_t k) const {
        return stems[k].sig < 0 ? pl->host[stems[k].cand].x : dry->i16 ? nullptr : dry->x[stems[k].sig];
    }
    // rendered from transient device copies: a host pool's banks and dry signals, a host or 16-bit dry pool's signals
    bool copied() const { return pl->host_res || (dry && dry->padded()); }
};
// A 16-bit signal's float32 expansion y[n] = x[n] / 32768, exact (x: device or mapped host memory)
__global__ void __launch_bounds__(256) k_expand_i16(const int16_t* __restrict__ x, float* __restrict__ y, long long N) {
    for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < N; n += (long long)gridDim.x * blockDim.x)
        y[n] = i16_sample(x[n]);
}
static int expand_i16(ss_ctx* c, const int16_t* x, float* y, long long N, cudaStream_t s) {
    const long long blocks = std::min((N + 255) / 256, (long long)c->sm_count * 8);
    k_expand_i16<<<(unsigned)blocks, 256, 0, s>>>(x, y, N);
    CK(cudaGetLastError());
    c->launches += 1;
    return SS_OK;
}
// every candidate of a pool with its own x, in candidate order (stem i is candidate i)
static StemSet own_stems(const ss_pool* pl) {
    StemSet S;
    S.pl = pl;
    for (int i = 0; i < pl->n; ++i) S.stems.push_back({i, -1});
    return S;
}

struct StemGroups {
    size_t cap = kLevelStemBytes;         // bytes of the transient buffer
    std::vector<int> first;               // group g holds stems [first[g], first[g + 1])
    std::vector<size_t> at;               // stem k's (C, N) output at byte at[k] of the buffer
};
static StemGroups stem_groups(const StemSet& S) {
    StemGroups G;
    const int n = (int)S.stems.size();
    for (int k = 0; k < n; ++k) G.cap = std::max(G.cap, align_up(4 * (size_t)S.pl->C * S.N(k), 256));
    G.first.assign(1, 0);
    G.at.resize(n);
    size_t used = 0;
    for (int k = 0; k < n; ++k) {
        const size_t b = align_up(4 * (size_t)S.pl->C * S.N(k), 256);
        if (used > 0 && used + b > G.cap) { G.first.push_back(k); used = 0; }
        G.at[k] = used;
        used += b;
    }
    G.first.push_back(n);
    return G;
}
// Render every group into `tmp` on `s` (after the pool's banks are complete), and after each group's render enqueue
// group(first, last) on `s`, whatever reads those stems before the next group overwrites them.  Returns when `s` is idle.
// Copied stems [first, first + n) (items, rendered whole): a host pool's reverberant spectra - once per run of
// consecutive stems of one candidate - and every stem's dry signal copied into transient device memory and rendered from
// there, in batches of at most kLevelStemBytes of copies (or one stem's, when larger), each behind the previous batch's
// render on `s`.  `buf` holds `cap` = stem_copy_cap bytes.  A tap-form pool's candidate is copied as its tap rows and
// rendered as a whole source with those RIRs (L = K * 4096, no flags): k_prepare then transforms the rows bank_build
// transforms for a spectral bank of the same RIRs, paired alike, into the same spectra.
static size_t stem_bank_bytes(const StemSet& S, size_t k) {
    const ss_bank* b = S.pl->banks[S.stems[k].cand];
    return S.pl->host_res ? align_up(S.pl->taps ? b->tap_bytes() : b->set_bytes(), 256) : 0;
}
static size_t stem_x_bytes(const StemSet& S, size_t k) { return align_up(sizeof(float) * (size_t)S.N(k), 256); }
static bool stem_new_bank(const StemSet& S, size_t k, bool batch_start) {
    return S.pl->host_res && (batch_start || S.stems[k - 1].cand != S.stems[k].cand);
}
static size_t stem_copy_cap(const StemSet& S) {
    size_t cap = 0, total = 0;
    for (size_t k = 0; k < S.stems.size(); ++k) {
        cap = std::max(cap, stem_bank_bytes(S, k) + stem_x_bytes(S, k));
        total += (stem_new_bank(S, k, k == 0) ? stem_bank_bytes(S, k) : 0) + stem_x_bytes(S, k);
    }
    return std::max(cap, std::min(total, kLevelStemBytes));
}
static int render_copied_stems(const StemSet& S, ss_source* items, int first, int n, char* buf, size_t cap,
                               cudaStream_t s) {
    std::vector<ss_bank> shells(n);
    for (int lo = 0; lo < n;) {
        size_t used = 0;
        int hi = lo;
        const ss_bank* shell = nullptr;
        const float* taps = nullptr;                    // (a tap-form pool) the candidate's copied rows
        for (; hi < n; ++hi) {
            const size_t k = (size_t)(first + hi);
            const bool new_bank = stem_new_bank(S, k, hi == lo);
            if (hi > lo && used + (new_bank ? stem_bank_bytes(S, k) : 0) + stem_x_bytes(S, k) > cap) break;
            if (new_bank && S.pl->taps) {
                const ss_bank* b = S.pl->banks[S.stems[k].cand];
                taps = (const float*)(buf + used);
                CK(cudaMemcpyAsync(buf + used, b->spec, b->tap_bytes(), cudaMemcpyDefault, s));
                used += stem_bank_bytes(S, k);
            } else if (new_bank) {
                const ss_bank* b = S.pl->banks[S.stems[k].cand];
                ss_bank& sh = shells[hi];
                sh = *b;                                // the bank's shape and `ready`, spectra from the copy
                sh.h_mem = nullptr; sh.d_mem = nullptr; sh.cut = nullptr; sh.spec = (float2*)(buf + used);
                CK(cudaMemcpyAsync(sh.spec, b->spec, b->set_bytes(), cudaMemcpyDefault, s));   // the reverberant set
                used += stem_bank_bytes(S, k);
                shell = &sh;
            }
            float* x = (float*)(buf + used);
            if (S.stems[k].sig >= 0 && S.dry->i16) {
                const int st = expand_i16(S.pl->c, S.dry->x16[S.stems[k].sig], x, S.N(k), s);
                if (st) return st;
            } else {
                CK(cudaMemcpyAsync(x, S.x(k), sizeof(float) * (size_t)S.N(k), cudaMemcpyDefault, s));
            }
            used += stem_x_bytes(S, k);
            items[hi].x = x;
            if (S.pl->taps) {
                items[hi].rir = taps; items[hi].rir_bank = nullptr; items[hi].L = S.pl->banks[S.stems[k].cand]->K * kB;
            } else if (S.pl->host_res) {
                items[hi].rir_bank = shell;
            }
        }
        const int st = ss_render_dev(S.pl->c, items + lo, hi - lo, (void*)s);   // the next batch's copies wait on `s`
        if (st) return st;
        lo = hi;
    }
    return SS_OK;
}
template <class Group>
static int render_stem_groups(const StemSet& S, const StemGroups& G, char* tmp, cudaStream_t s, Group group) {
    const ss_pool* pl = S.pl;
    CK(cudaStreamWaitEvent(s, pl->ready, 0));           // banks may still be building
    char* copies = nullptr;                             // transient copies of banks and dry signals
    const size_t copy_cap = S.copied() ? stem_copy_cap(S) : 0;
    if (S.copied()) CK(cudaMalloc((void**)&copies, copy_cap));
    struct Free { char* p; ~Free() { if (p) cudaFree(p); } } free_copies{copies};   // (cudaFree waits for the device)
    std::vector<ss_source> items;
    for (size_t g = 0; g + 1 < G.first.size(); ++g) {
        items.clear();
        for (int k = G.first[g]; k < G.first[g + 1]; ++k) {
            const int i = S.stems[k].cand;
            const PoolEntry& e = pl->host[i];
            ss_source it; memset(&it, 0, sizeof(it));
            it.x = S.x(k); it.out = (float*)(tmp + G.at[k]); it.N = e.N; it.P = e.P; it.C = pl->C; it.L = pl->banks[i]->L;
            it.mode = pl->mode; it.rir_bank = pl->banks[i];
            if (pl->mode == SS_MOVING_BOUNDS) { it.bounds = e.bounds; it.bounds_host = pl->bounds_host.data() + pl->bounds_off[i]; }
            items.push_back(it);
        }
        int st = S.copied() ? render_copied_stems(S, items.data(), G.first[g], (int)items.size(), copies, copy_cap, s)
                            : ss_render_dev(pl->c, items.data(), (int)items.size(), (void*)s);   // the next group waits on `s`
        if (st == SS_OK) st = group(G.first[g], G.first[g + 1]);
        if (st) return st;
    }
    CK(cudaStreamSynchronize(s));
    return SS_OK;
}
// One transient stream per build call, synchronised and destroyed on every return path
struct BuildStream {
    cudaStream_t s = nullptr;
    ~BuildStream() { if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); } }
};

// ----------------------------------------------------------------------------- loudness gains of a pool
// Device memory of one loudness build (ss_pool_loudness, ss_pair_gains_create): the gating tables of the measured
// candidates (post[i]: candidate i's gating plan; one copy per distinct set of host arrays), every stem's result, and
// one group's scratch.  entry(k, q) fills q with stem k's entry - its candidate's plan and its target - and returns
// whether stem k is measured.  res receives (LUFS, gain) per stem, in stem order.
template <class Entry>
static int loudness_build(const StemSet& S, const ss_post_lufs* post, Entry entry, cudaStream_t s,
                          std::vector<void*>& owned, std::vector<double>& res) {
    const ss_pool* pl = S.pl;
    const size_t n = S.stems.size();
    const GatingTables tabs = gating_tables(post, pl->n);
    const StemGroups G = stem_groups(S);
    ss_post_lufs q;
    size_t scratch = 0;                                 // the largest group's loudness scratch
    for (size_t g = 0; g + 1 < G.first.size(); ++g) {
        size_t b = 0;
        for (int k = G.first[g]; k < G.first[g + 1]; ++k)
            if (entry(k, q)) b += loud_scratch_bytes(q, pl->C);
        scratch = std::max(scratch, b);
    }
    char *d_tab = nullptr, *d_scr = nullptr, *tmp = nullptr;
    double* d_res = nullptr;
    CK(cudaMalloc((void**)&d_tab, std::max(tabs.bytes.size(), (size_t)256))); owned.push_back(d_tab);
    CK(cudaMalloc((void**)&d_res, 2 * sizeof(double) * n)); owned.push_back(d_res);
    CK(cudaMalloc((void**)&d_scr, std::max(scratch, (size_t)256))); owned.push_back(d_scr);
    CK(cudaMalloc((void**)&tmp, G.cap)); owned.push_back(tmp);
    if (!tabs.bytes.empty()) CK(cudaMemcpy(d_tab, tabs.bytes.data(), tabs.bytes.size(), cudaMemcpyHostToDevice));
    std::vector<ss_loud_item> li;
    const int st = render_stem_groups(S, G, tmp, s, [&](int first, int last) -> int {
        // every measured stem of the group: the launches of ss_loudness_dev on its (C, N) output, measure only
        li.clear();
        char* scr = d_scr;
        for (int k = first; k < last; ++k) {
            if (!entry(k, q)) continue;
            const int i = S.stems[k].cand;
            li.push_back(loud_item(q, d_tab + tabs.at[i], (const float*)(tmp + G.at[k]), nullptr, pl->host[i].N, pl->C,
                                   (double*)scr, d_res + 2 * (size_t)k));
            scr += loud_scratch_bytes(q, pl->C);
        }
        for (size_t k = 0; k < li.size(); k += 65535) {   // ss_loudness_dev's item limit
            const int st2 = ss_loudness_dev(pl->c, li.data() + k, (int)std::min(li.size() - k, (size_t)65535), (void*)s);
            if (st2) return st2;
        }
        return SS_OK;
    });
    if (st) return st;
    res.resize(2 * n);
    CK(cudaMemcpy(res.data(), d_res, 2 * sizeof(double) * n, cudaMemcpyDeviceToHost));
    return SS_OK;
}

extern "C" int ss_pool_loudness(ss_pool* pl, const ss_post_lufs* post) {
    if (!pl || !post) return SS_ERR_INVALID;
    if (pl->C > 8) return SS_ERR_UNSUPPORTED;           // as ss_loudness_dev
    if (pl->gains || pl->levels || pl->planned || check_post_lufs(post, pl->n)) return SS_ERR_INVALID;
    CK(cudaSetDevice(pl->c->device));
    std::vector<void*> owned;
    std::vector<double> res;
    int st;
    {
        BuildStream bs;
        CK(cudaStreamCreateWithFlags(&bs.s, cudaStreamNonBlocking));
        st = loudness_build(own_stems(pl), post, [&](int i, ss_post_lufs& q) { q = post[i]; return post[i].brk != nullptr; },
                            bs.s, owned, res);
    }
    for (void* q : owned) cudaFree(q);
    if (st != SS_OK) return st;                         // no gains: the pool is as it was
    const int n = pl->n;
    std::vector<float> g(n, 1.0f);
    std::vector<double> loud(2 * (size_t)n, NAN);
    for (int i = 0; i < n; ++i) {
        if (!post[i].brk) continue;
        loud[2 * i] = res[2 * i]; loud[2 * i + 1] = res[2 * i + 1];
        g[i] = (float)res[2 * i + 1];                   // what k_loud_scale multiplies by
    }
    float* d_g = nullptr;
    CK(cudaMalloc((void**)&d_g, sizeof(float) * (size_t)n));
    const cudaError_t e = cudaMemcpy(d_g, g.data(), sizeof(float) * (size_t)n, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(d_g); g_last_cuda = (int)e; return SS_ERR_CUDA; }
    pl->gains = d_g;
    pl->loud.swap(loud);
    for (int i = 0; i < n; ++i)
        if (post[i].brk && post[i].result) { post[i].result[0] = res[2 * i]; post[i].result[1] = res[2 * i + 1]; }
    return SS_OK;
}

// ----------------------------------------------------------------------------- level tables of a pool
// k_levels turns each group of whole stems into its tables; a pool with gains first scales each stem by its candidate's
// (float)gain with k_loud_scale itself, so that the tables describe the normalised stems its slots render.
static int levels_build(ss_pool* pl, bool mono, cudaStream_t s, std::vector<void*>& owned) {
    const int n = pl->n;
    pl->level_off.assign(n + 1, 0);
    for (int i = 0; i < n; ++i) pl->level_off[i + 1] = pl->level_off[i] + pl->host[i].N + 1;
    if (pl->host_res) {                                 // a host pool: k_levels writes and k_draw reads them over PCIe
        CK(cudaHostAlloc((void**)&pl->h_levels, level_bytes(pl), cudaHostAllocMapped | cudaHostAllocPortable));
        CK(cudaHostGetDevicePointer((void**)&pl->levels, pl->h_levels, 0));
    } else {
        CK(cudaMalloc((void**)&pl->levels, level_bytes(pl)));
    }
    CK(cudaMalloc((void**)&pl->level_ptr, sizeof(double*) * (size_t)n));
    std::vector<const double*> ptr(n);
    for (int i = 0; i < n; ++i) ptr[i] = pl->levels + pl->level_off[i];
    CK(cudaMemcpy(pl->level_ptr, ptr.data(), sizeof(double*) * (size_t)n, cudaMemcpyHostToDevice));
    const StemSet S = own_stems(pl);
    const StemGroups G = stem_groups(S);
    char* tmp = nullptr;
    LevelItem* d_items = nullptr;
    double* d_res = nullptr;                            // the (LUFS, gain) pairs k_loud_scale reads its gain from
    CK(cudaMalloc((void**)&tmp, G.cap)); owned.push_back(tmp);
    std::vector<LevelItem> li(n);
    for (int i = 0; i < n; ++i) li[i] = {(const float*)(tmp + G.at[i]), pl->levels + pl->level_off[i], pl->host[i].N, pl->C, 0};
    CK(cudaMalloc((void**)&d_items, sizeof(LevelItem) * (size_t)n)); owned.push_back(d_items);
    CK(cudaMemcpy(d_items, li.data(), sizeof(LevelItem) * (size_t)n, cudaMemcpyHostToDevice));
    if (pl->gains) {
        std::vector<double> r(pl->loud);
        for (int i = 0; i < n; ++i) if (isnan(r[2 * i + 1])) r[2 * i + 1] = 1.0;      // unmeasured: gain 1
        CK(cudaMalloc((void**)&d_res, sizeof(double) * r.size())); owned.push_back(d_res);
        CK(cudaMemcpy(d_res, r.data(), sizeof(double) * r.size(), cudaMemcpyHostToDevice));
    }
    std::vector<ScaleItem> sc;
    return render_stem_groups(S, G, tmp, s, [&](int first, int last) -> int {
        if (d_res) {
            sc.clear();
            for (int i = first; i < last; ++i) sc.push_back(ScaleItem{(float*)li[i].y, d_res + 2 * (size_t)i, pl->host[i].N, pl->C});
            for (size_t k = 0; k < sc.size(); k += 65535) {   // one gridDim.y row per stem
                const int st = loud_scale_dev(pl->c, sc.data() + k, (int)std::min(sc.size() - k, (size_t)65535), s);
                if (st) return st;
            }
        }
        return levels_enqueue(pl->c, d_items + first, last - first, mono, s);
    });
}

extern "C" int ss_pool_levels(ss_pool* pl, uint32_t flags) {
    if (!pl || (flags & ~SS_MIX_MONO) || pl->level_flags >= 0 || pl->levels) return SS_ERR_INVALID;
    CK(cudaSetDevice(pl->c->device));
    std::vector<void*> owned;
    int st;
    {
        BuildStream bs;
        CK(cudaStreamCreateWithFlags(&bs.s, cudaStreamNonBlocking));
        st = levels_build(pl, (flags & SS_MIX_MONO) != 0, bs.s, owned);
    }
    for (void* q : owned) cudaFree(q);
    if (st != SS_OK) {                                  // no tables: the pool is as it was
        free_levels(pl);
        return st;
    }
    pl->level_flags = (int)flags;
    return SS_OK;
}

// ----------------------------------------------------------------------------- dry pools
extern "C" void ss_dry_pool_destroy(ss_dry_pool* dp) {
    if (!dp) return;
    cudaSetDevice(dp->c->device);
    cudaDeviceSynchronize();                            // (a plan that used it may run on any stream)
    if (dp->ptrs) cudaFree(dp->ptrs);
    if (dp->h_levels) cudaFreeHost(dp->h_levels); else if (dp->levels) cudaFree(dp->levels);
    if (dp->level_ptr && !dp->i16) cudaFree(dp->level_ptr);   // (a 16-bit pool's lie in ptrs)
    if (dp->h_x) cudaFreeHost(dp->h_x);
    if (dp->d_x) cudaFree(dp->d_x);
    delete dp;
}
static int64_t dry_level_bytes(const ss_dry_pool* dp) {
    return dp->levels ? (int64_t)sizeof(double) * dp->level_off[dp->n] : 0;
}
extern "C" int64_t ss_dry_pool_bytes(const ss_dry_pool* dp) {
    if (!dp) return 0;
    int64_t b = (int64_t)sizeof(float*) * dp->n + (int64_t)dp->d_x_bytes;
    if (dp->levels) b += (dp->host ? 0 : dry_level_bytes(dp)) + (int64_t)sizeof(double*) * dp->n;
    return b;
}
extern "C" int64_t ss_dry_pool_host_bytes(const ss_dry_pool* dp) {
    return dp && dp->host ? (int64_t)dp->h_x_bytes + dry_level_bytes(dp) : 0;
}
extern "C" const double* ss_dry_pool_level_table(const ss_dry_pool* dp, int i) {
    if (!dp || !dp->levels || i < 0 || i >= dp->n) return nullptr;
    return (dp->host ? dp->h_levels : dp->levels) + dp->level_off[i];
}
extern "C" int ss_dry_pool_level_stride(const ss_dry_pool* dp) { return dp ? dp->stride() : 0; }
extern "C" const int16_t* ss_dry_pool_signal_i16(const ss_dry_pool* dp, int i) {
    if (!dp || !dp->i16 || i < 0 || i >= dp->n) return nullptr;
    return dp->host ? (const int16_t*)(dp->h_x + ((const char*)dp->x16[i] - (const char*)dp->x16[0])) : dp->x16[i];
}
// A 16-bit dry pool: the signals into its arena (device memory, or pinned, mapped host memory with SS_DRY_HOST), each at
// a 64-byte boundary and zero-padded to the next (k_stage reads whole groups of 4 samples around a read set); x16[i]
// receives the signal's device (or mapped device) address
static int dry_i16_copies(ss_dry_pool* dp, const int16_t* const* x) {
    const int n = dp->n;
    std::vector<size_t> xo(n + 1, 0);
    for (int i = 0; i < n; ++i) xo[i + 1] = xo[i] + align_up(sizeof(int16_t) * (size_t)dp->N[i], 64);
    char* dx = nullptr;
    if (dp->host) {
        dp->h_x_bytes = xo[n];
        CK(cudaHostAlloc((void**)&dp->h_x, dp->h_x_bytes, cudaHostAllocMapped | cudaHostAllocPortable));
        CK(cudaHostGetDevicePointer((void**)&dx, dp->h_x, 0));
    } else {
        dp->d_x_bytes = xo[n];
        CK(cudaMalloc((void**)&dp->d_x, dp->d_x_bytes));
        CK(cudaMemset(dp->d_x, 0, dp->d_x_bytes));
        dx = dp->d_x;
    }
    dp->x16.resize(n);
    for (int i = 0; i < n; ++i) {
        const size_t b = sizeof(int16_t) * (size_t)dp->N[i];
        CK(cudaMemcpy((dp->host ? dp->h_x : dp->d_x) + xo[i], x[i], b, cudaMemcpyDefault));
        if (dp->host) memset(dp->h_x + xo[i] + b, 0, xo[i + 1] - xo[i] - b);
        dp->x16[i] = (const int16_t*)(dx + xo[i]);
    }
    return SS_OK;
}
// A 16-bit pool's sparse tables from full ones: q[j] = Q[min(64 j, N)], j = 0..ceil(N / 64)
__global__ void __launch_bounds__(256) k_level_sample(const double* __restrict__ Q, double* __restrict__ q, long long N) {
    const long long m = (N + kLevelStride - 1) / kLevelStride;
    for (long long j = (long long)blockIdx.x * blockDim.x + threadIdx.x; j <= m; j += (long long)gridDim.x * blockDim.x)
        q[j] = Q[j * kLevelStride < N ? j * kLevelStride : N];
}
// A host dry pool: the signals into its pinned, mapped arena, each at a 64-byte boundary and zero-padded to whole
// float4s (k_stage copies whole float4s around a read set); x[i] becomes the signal's mapped device address
static int dry_host_copies(ss_dry_pool* dp) {
    const int n = dp->n;
    std::vector<size_t> xo(n + 1, 0);
    for (int i = 0; i < n; ++i) xo[i + 1] = xo[i] + align_up(sizeof(float) * (size_t)dp->N[i], 64);
    dp->h_x_bytes = xo[n];
    CK(cudaHostAlloc((void**)&dp->h_x, dp->h_x_bytes, cudaHostAllocMapped | cudaHostAllocPortable));
    char* dx = nullptr;
    CK(cudaHostGetDevicePointer((void**)&dx, dp->h_x, 0));
    for (int i = 0; i < n; ++i) {
        const size_t b = sizeof(float) * (size_t)dp->N[i];
        CK(cudaMemcpy(dp->h_x + xo[i], dp->x[i], b, cudaMemcpyDefault));
        memset(dp->h_x + xo[i] + b, 0, xo[i + 1] - xo[i] - b);
        dp->x[i] = (const float*)(dx + xo[i]);
    }
    return SS_OK;
}
// The level tables of a host or 16-bit dry pool: k_levels over transient device copies of the signals (a 16-bit pool's:
// their float32 expansions), in batches of at most kLevelStemBytes of copies (or one signal's, when larger), each
// batch's copies behind the previous batch's scan on `s`.  k_levels writes a host dry pool's tables into pinned, mapped
// host memory; a 16-bit pool's full tables go to transient device memory too, and k_level_sample keeps every 64th entry
// and the last in the pool's tables, which are therefore the float pool's entries bit for bit.  `li` holds every
// signal's descriptor with its table.
static int dry_copied_levels(ss_dry_pool* dp, std::vector<LevelItem>& li, cudaStream_t s) {
    const int n = dp->n;
    std::vector<size_t> at(n), tat(n);
    std::vector<int> first(1, 0);
    size_t used = 0, cap = kLevelStemBytes, tused = 0, tcap = 0;
    for (int i = 0; i < n; ++i) cap = std::max(cap, align_up(sizeof(float) * (size_t)dp->N[i], 256));
    for (int i = 0; i < n; ++i) {
        const size_t b = align_up(sizeof(float) * (size_t)dp->N[i], 256);
        if (used > 0 && used + b > cap) { first.push_back(i); used = 0; tused = 0; }
        at[i] = used;
        used += b;
        tat[i] = tused;                                 // (a 16-bit pool: the signal's full table in the batch's)
        tused += align_up(sizeof(double) * ((size_t)dp->N[i] + 1), 256);
        tcap = std::max(tcap, tused);
    }
    first.push_back(n);
    if (first.size() == 2) cap = used;                  // one batch: no more than it needs
    char *buf = nullptr, *tabs = nullptr;
    CK(cudaMalloc((void**)&buf, cap));
    struct Free { void* p; ~Free() { if (p) cudaFree(p); } } free_buf{buf};   // (cudaFree waits for the device)
    if (dp->i16) CK(cudaMalloc((void**)&tabs, tcap));
    struct Free free_tabs{tabs};
    std::vector<double*> q(n);                          // the pool's tables
    for (int i = 0; i < n; ++i) {
        q[i] = li[i].q;
        li[i].y = (const float*)(buf + at[i]);
        if (dp->i16) li[i].q = (double*)(tabs + tat[i]);
    }
    LevelItem* d_items = nullptr;
    CK(cudaMalloc((void**)&d_items, sizeof(LevelItem) * (size_t)n));
    struct Free free_items{d_items};
    CK(cudaMemcpy(d_items, li.data(), sizeof(LevelItem) * (size_t)n, cudaMemcpyHostToDevice));
    for (size_t g = 0; g + 1 < first.size(); ++g) {
        for (int i = first[g]; i < first[g + 1]; ++i) {
            if (dp->i16) {
                const int st = expand_i16(dp->c, dp->x16[i], (float*)li[i].y, dp->N[i], s);
                if (st) return st;
            } else {
                CK(cudaMemcpyAsync((void*)li[i].y, dp->x[i], sizeof(float) * (size_t)dp->N[i], cudaMemcpyDefault, s));
            }
        }
        for (int k = first[g]; k < first[g + 1]; k += 65535) {
            const int st = levels_enqueue(dp->c, d_items + k, std::min(first[g + 1] - k, 65535), true, s);
            if (st) return st;
        }
        if (dp->i16)
            for (int i = first[g]; i < first[g + 1]; ++i) {
                const long long m = ((long long)dp->N[i] + kLevelStride - 1) / kLevelStride + 1;
                k_level_sample<<<(unsigned)std::min((m + 255) / 256, (long long)dp->c->sm_count * 8), 256, 0, s>>>(
                    li[i].q, q[i], dp->N[i]);
                CK(cudaGetLastError());
                dp->c->launches += 1;
            }
    }
    CK(cudaStreamSynchronize(s));
    return SS_OK;
}
// The signals' pointer array (a host dry pool's after its arena copies), and with level tables the tables - k_levels over
// each signal as a one-channel stem, whose mono fold is the signal itself - built on a transient stream; returns when
// they are complete.
static int dry_pool_build(ss_dry_pool* dp, bool levels) {
    const int n = dp->n;
    if (dp->host && !dp->i16) { const int st = dry_host_copies(dp); if (st) return st; }
    // the signal pointers, and a 16-bit pool's table pointers behind them
    const size_t n_ptr = (dp->i16 && levels ? 2 : 1) * (size_t)n;
    CK(cudaMalloc((void**)&dp->ptrs, sizeof(float*) * n_ptr));
    if (dp->i16) CK(cudaMemcpy(dp->ptrs, dp->x16.data(), sizeof(int16_t*) * (size_t)n, cudaMemcpyHostToDevice));
    else CK(cudaMemcpy(dp->ptrs, dp->x.data(), sizeof(float*) * (size_t)n, cudaMemcpyHostToDevice));
    if (!levels) return SS_OK;
    dp->level_off.assign(n + 1, 0);
    const int r = dp->stride();
    for (int i = 0; i < n; ++i) dp->level_off[i + 1] = dp->level_off[i] + (dp->N[i] + r - 1) / r + 1;
    const size_t tb = sizeof(double) * (size_t)dp->level_off[n];
    if (dp->host) {                                     // k_levels writes and k_draw reads them over PCIe
        CK(cudaHostAlloc((void**)&dp->h_levels, tb, cudaHostAllocMapped | cudaHostAllocPortable));
        CK(cudaHostGetDevicePointer((void**)&dp->levels, dp->h_levels, 0));
    } else {
        CK(cudaMalloc((void**)&dp->levels, tb));
    }
    if (dp->i16) dp->level_ptr = (const double**)(dp->ptrs + n);
    else CK(cudaMalloc((void**)&dp->level_ptr, sizeof(double*) * (size_t)n));
    std::vector<const double*> ptr(n);
    std::vector<LevelItem> li(n);
    for (int i = 0; i < n; ++i) {
        ptr[i] = dp->levels + dp->level_off[i];
        li[i] = {dp->i16 ? nullptr : dp->x[i], dp->levels + dp->level_off[i], dp->N[i], 1, 0};
    }
    CK(cudaMemcpy(dp->level_ptr, ptr.data(), sizeof(double*) * (size_t)n, cudaMemcpyHostToDevice));
    BuildStream bs;
    CK(cudaStreamCreateWithFlags(&bs.s, cudaStreamNonBlocking));
    if (dp->padded()) return dry_copied_levels(dp, li, bs.s);
    LevelItem* d_items = nullptr;
    CK(cudaMalloc((void**)&d_items, sizeof(LevelItem) * (size_t)n));
    struct Free { void* p; ~Free() { cudaFree(p); } } free_items{d_items};   // (cudaFree waits for the device)
    CK(cudaMemcpy(d_items, li.data(), sizeof(LevelItem) * (size_t)n, cudaMemcpyHostToDevice));
    for (int k = 0; k < n; k += 65535) {
        const int st = levels_enqueue(dp->c, d_items + k, std::min(n - k, 65535), true, bs.s);
        if (st) return st;
    }
    CK(cudaStreamSynchronize(bs.s));
    return SS_OK;
}
extern "C" int ss_dry_pool_create(ss_ctx* c, const float* const* x, const int32_t* lengths, int n, uint32_t flags,
                                  ss_dry_pool** out) {
    if (!c || !x || !lengths || !out || n < 1 || n > (1 << 24) || (flags & ~(SS_DRY_LEVELS | SS_DRY_HOST)))
        return SS_ERR_INVALID;
    *out = nullptr;
    for (int i = 0; i < n; ++i)                         // (the bound of validate_item on N)
        if (!x[i] || ((uintptr_t)x[i] & 3) || lengths[i] < 1 || lengths[i] > 0x7fffffff - 2 * kF) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    ss_dry_pool* dp = new (std::nothrow) ss_dry_pool();
    if (!dp) return SS_ERR_NOMEM;
    dp->c = c; dp->n = n; dp->host = (flags & SS_DRY_HOST) != 0;
    dp->x.assign(x, x + n);
    dp->N.assign(lengths, lengths + n);
    dp->n_min = *std::min_element(lengths, lengths + n);
    const int st = dry_pool_build(dp, (flags & SS_DRY_LEVELS) != 0);
    if (st != SS_OK) { ss_dry_pool_destroy(dp); return st; }
    *out = dp;
    return SS_OK;
}
extern "C" int ss_dry_pool_create_i16(ss_ctx* c, const int16_t* const* x, const int32_t* lengths, int n, uint32_t flags,
                                      ss_dry_pool** out) {
    if (!c || !x || !lengths || !out || n < 1 || n > (1 << 24) || (flags & ~(SS_DRY_LEVELS | SS_DRY_HOST)))
        return SS_ERR_INVALID;
    *out = nullptr;
    for (int i = 0; i < n; ++i) if (!x[i] || ((uintptr_t)x[i] & 1)) return SS_ERR_INVALID;
    for (int i = 0; i < n; ++i)                         // (beyond 2^23 samples a table's sums need not be exact)
        if (lengths[i] < 1 || lengths[i] > (1 << 23)) return SS_ERR_UNSUPPORTED;
    CK(cudaSetDevice(c->device));
    ss_dry_pool* dp = new (std::nothrow) ss_dry_pool();
    if (!dp) return SS_ERR_NOMEM;
    dp->c = c; dp->n = n; dp->host = (flags & SS_DRY_HOST) != 0; dp->i16 = true;
    dp->N.assign(lengths, lengths + n);
    dp->n_min = *std::min_element(lengths, lengths + n);
    int st = dry_i16_copies(dp, x);
    if (st == SS_OK) st = dry_pool_build(dp, (flags & SS_DRY_LEVELS) != 0);
    if (st != SS_OK) { ss_dry_pool_destroy(dp); return st; }
    *out = dp;
    return SS_OK;
}

// ----------------------------------------------------------------------------- pair gains
// The (float)gain of every (dry signal d, candidate i) pair of a pool and a dry pool, at [d * n + i] in device memory,
// which dry-picked slots take in place of their candidate's gain (pair_table).  The pools are kept only to check that a
// plan's slot names the pool and the dry pool the table was measured over.
constexpr int64_t kMaxPairs = 1 << 26;
struct ss_pair_gains {
    ss_ctx* c = nullptr;
    const ss_pool* pool = nullptr;
    const ss_dry_pool* dry = nullptr;
    float* gains = nullptr;
    int64_t pairs = 0;
};
extern "C" void ss_pair_gains_destroy(ss_pair_gains* g) {
    if (!g) return;
    cudaSetDevice(g->c->device);
    cudaDeviceSynchronize();                            // (a plan that used it may run on any stream)
    if (g->gains) cudaFree(g->gains);
    delete g;
}
extern "C" int64_t ss_pair_gains_bytes(const ss_pair_gains* g) { return g ? (int64_t)sizeof(float) * g->pairs : 0; }
extern "C" int ss_pair_gains_create(ss_ctx* c, const ss_pool* pl, const ss_dry_pool* dp, const ss_post_lufs* post,
                                    const double* targets, double* results, ss_pair_gains** out) {
    if (!c || !pl || !dp || !post || !targets || !out || pl->c != c || dp->c != c) return SS_ERR_INVALID;
    if (pl->C > 8) return SS_ERR_UNSUPPORTED;           // as ss_loudness_dev
    const int n = pl->n;
    const int64_t pairs = (int64_t)dp->n * n;
    if (pairs > kMaxPairs) return SS_ERR_UNSUPPORTED;
    for (const PoolEntry& e : pl->host) if (e.N > dp->n_min) return SS_ERR_INVALID;   // (ss_plan_create_dry's rule)
    if (check_post_lufs(post, n)) return SS_ERR_INVALID;
    for (int64_t k = 0; k < pairs; ++k) if (!isnan(targets[k]) && !isfinite(targets[k])) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    // the measured pairs, candidate-major: a host pool's bank is copied once per batch of its pairs
    StemSet S;
    S.pl = pl; S.dry = dp;
    for (int i = 0; i < n; ++i)
        if (post[i].brk)
            for (int d = 0; d < dp->n; ++d) if (!isnan(targets[(int64_t)d * n + i])) S.stems.push_back({i, d});
    std::vector<void*> owned;
    std::vector<double> res;
    int st = SS_OK;
    if (!S.stems.empty()) {
        BuildStream bs;
        CK(cudaStreamCreateWithFlags(&bs.s, cudaStreamNonBlocking));
        st = loudness_build(S, post, [&](int k, ss_post_lufs& q) {
            q = post[S.stems[k].cand];
            q.target_lufs = targets[(int64_t)S.stems[k].sig * n + S.stems[k].cand];
            return true;
        }, bs.s, owned, res);
    }
    for (void* q : owned) cudaFree(q);
    if (st != SS_OK) return st;
    std::vector<float> g((size_t)pairs, 1.0f);
    for (size_t k = 0; k < S.stems.size(); ++k)
        g[(size_t)S.stems[k].sig * n + S.stems[k].cand] = (float)res[2 * k + 1];   // what k_loud_scale multiplies by
    ss_pair_gains* pg = new (std::nothrow) ss_pair_gains();
    if (!pg) return SS_ERR_NOMEM;
    pg->c = c; pg->pool = pl; pg->dry = dp; pg->pairs = pairs;
    cudaError_t e = cudaMalloc((void**)&pg->gains, sizeof(float) * (size_t)pairs);
    if (e == cudaSuccess) e = cudaMemcpy(pg->gains, g.data(), sizeof(float) * (size_t)pairs, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { ss_pair_gains_destroy(pg); g_last_cuda = (int)e; return SS_ERR_CUDA; }
    if (results) {
        std::fill(results, results + 2 * pairs, (double)NAN);
        for (size_t k = 0; k < S.stems.size(); ++k) {
            double* const r = results + 2 * ((int64_t)S.stems[k].sig * n + S.stems[k].cand);
            r[0] = res[2 * k]; r[1] = res[2 * k + 1];
        }
    }
    *out = pg;
    return SS_OK;
}

// ----------------------------------------------------------------------------- plans (device path)
// A batch of device-resident sources bound once: validation, chunking, block tables and descriptor blocks are done at
// creation and stay resident in device memory together with the plan's own scratch, so a run is kernel launches only -
// captured into a CUDA graph on the first run (fork onto the context's internal streams, join back), one
// cudaGraphLaunch per run afterwards instead of ~25 runtime calls.  The pointers in `items` (and the contents of
// bounds_host) must stay valid and unchanged for the plan's life; buffer *contents* may change between runs.
struct DrawDesc;
struct StageSlot;
struct ss_plan {
    ss_ctx* c = nullptr;
    std::vector<ChunkLaunch> chunks;
    char* d_desc = nullptr;
    char* d_scratch[ss_ctx::kAux] = {};
    cudaGraphExec_t exec = nullptr;
    bool graph_failed = false;
    int launches_per_run = 0;
    // fork / join events of the plan's own (events recorded while capturing must not be waited on outside the graph,
    // which the context's events are)
    cudaEvent_t ev_fork = nullptr, ev_join[ss_ctx::kAux] = {};
    cudaStream_t s_cap = nullptr;      // capture origin: the caller's stream may be the legacy default stream, which cannot capture
    std::vector<ss_bank*> banks;       // banks of the plan's sources: every run waits for their construction
    std::vector<ss_pool*> pools;       // pools of its pooled slots: every run waits for each pool's `ready` event
    const MixItem* d_mix = nullptr;   // the mixtures' descriptors, in d_desc behind the chunk descriptors
    int n_mix = 0;
    bool mix_direct = false;           // some mixture has a dereverberation target: k_mix_write<true>
    const DrawDesc* d_draw = nullptr;  // the start draws' descriptors (k_draw), in d_desc behind the mixture scratch
    int n_draw = 0;
    const StageSlot* d_stage = nullptr;   // the staged slots' k_stage descriptors, in d_desc behind the draws
    int n_stage = 0;
    bool draw16 = false, stage16 = false; // a draw speaker / a staged slot has a 16-bit dry pick: k_draw<true> / k_stage<true>
    bool draw_stream = false, stage_stream = false;   // a draw speaker / a staged slot is a stream slot (STREAM)
    bool stage_bg = false;                            // a staged slot is a bed slot (k_stage<true, TAPS, true, true>)
    // slots of tap-form pools: k_stage<I16, true> reads d_taps (n_stage entries) and writes n_tap transform Sources
    // (d_tap_src, CTA ranges d_tap_prefix), which one k_prepare<false> of tap_ctas CTAs transforms behind it
    const StageTap* d_taps = nullptr;
    const Source* d_tap_src = nullptr;
    const int* d_tap_prefix = nullptr;
    int n_tap = 0, tap_ctas = 0;
    // loudness slots (ss_stream_lufs): their measuring descriptors (k_kweight, k_kw_scan, k_loud_gate<true>) and work-item
    // offsets, and their crops (k_loud_crop), in d_desc
    const LoudItem* d_loud = nullptr;
    const int* d_loud_prefix = nullptr;
    const LoudCrop* d_crop = nullptr;
    int n_loud = 0, loud_total = 0, crop_ctas = 0;
    double loud_rate = 0;
    // layout draws (ss_layout_draw): their descriptors (k_layout) in d_desc, and the dynamic shared memory of the most
    // scratch any of them needs
    const LayoutDesc* d_layout = nullptr;
    int n_layout = 0, layout_smem = 0;
    // with grouped layout draws (ss_layout_group): one LayoutGroup per layout draw (k_layout_grouped), or null
    const LayoutGroup* d_layout_group = nullptr;
    // value draws (ss_value_draw): their descriptors (k_values) in d_desc, and the rows every one of them has
    const ValueDesc* d_value = nullptr;
    int n_value = 0, value_rows = 0;
};

// ----------------------------------------------------------------------------- k_draw
// Crop start draws of a plan (ss_plan_draw).  A reader is a pooled slot whose win_start_dev is the draw's start; the
// speakers are readers with level tables: their pool's, or their dry pool's for a dry-picked speaker (speaker_table).  The
// picks are clamped as k_blocks clamps them (which reports bits 3 and 4).
constexpr int kDrawReaders = 16, kDrawSpeakers = 8, kDrawTries = 4096, kMaxDraws = 65535;
struct DrawReader {
    const PoolEntry* pool;            // the slot's pool table ...
    const int* pick;                  // ... and pick
    const double* const* levels;      // the pool's level table pointers (speakers without a dry pick), else null
    int n;                            // candidates in the pool
    double D;                         // elements of one crop in a table: len (mono or dry) or C * len
    const double* const* dry_levels;  // a dry-picked speaker: its dry pool's table pointers, else null ...
    const int* dry_pick;              // ... its dry pick ...
    int n_dry;                        // ... and the dry pool's signal count
    int dry16;                        // 1: the dry pool is 16-bit (sparse tables, speaker_signal_i16; k_draw<true> only)
                                      // 2: a stream slot (k_draw<true, true> only): dry_pick holds its DryStream
};
static_assert(sizeof(DrawReader) == 64, "DrawReader layout");
struct DrawDesc {
    int* start;
    const double* u;
    int* used;
    int tries, len, n_readers, S;
    float threshold_db;
    int spk[kDrawSpeakers];           // speaker k is reader spk[k]
    DrawReader r[kDrawReaders];
};

// One warp per draw: the readers' picked N give M (a lane per reader), then 32 tries at a time, a lane per try, and a
// ballot takes the first try at which no speaker is silent; after the last try without one, the last try's start.
// k_draw<true> (a plan with a 16-bit dry-picked speaker) tests such a speaker from its sparse table and its signal's
// samples (draw_silent_i16): at most 2 * 63 samples and two table entries per try, over PCIe for a host pool.
// k_draw<true, true> (a plan with a stream speaker) tests such a speaker by walking its layout at every try
// (draw_silent_stream): the layout's entries are the same for every lane, the utterances' samples per lane.
template <bool I16, bool STREAM = false>
__global__ void __launch_bounds__(128) k_draw(const DrawDesc* __restrict__ draws, int n) {
    const int lane = threadIdx.x & 31, di = blockIdx.x * 4 + (threadIdx.x >> 5);
    if (di >= n) return;
    const DrawDesc& d = draws[di];
    bool bad;
    int M = 0x7fffffff;
    if (lane < d.n_readers) {
        const DrawReader& r = d.r[lane];
        M = draw_span(r.pool[clamp_pick(*r.pick, r.n, bad)].N, d.len);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) M = min(M, __shfl_xor_sync(0xffffffffu, M, o));
    const double* Q[kDrawSpeakers];
    double D[kDrawSpeakers];
    const int16_t* X[kDrawSpeakers];                    // (k_draw<true>) a 16-bit speaker's signal, else null
    const DryStream* W[kDrawSpeakers];                  // (k_draw<true, true>) a stream speaker's layout, else null
#pragma unroll
    for (int k = 0; k < kDrawSpeakers; ++k) {
        Q[k] = nullptr; D[k] = 1.0; X[k] = nullptr; W[k] = nullptr;
        if (k < d.S) {
            const DrawReader& r = d.r[d.spk[k]];
            if (STREAM && r.dry16 == 2) { W[k] = reinterpret_cast<const DryStream*>(r.dry_pick); continue; }
            Q[k] = speaker_table(r.levels, r.pick, r.n, r.dry_levels, r.dry_pick, r.n_dry);
            D[k] = r.D;
            if (I16 && r.dry16) X[k] = speaker_signal_i16(r.dry_levels, r.dry_pick, r.n_dry);
        }
    }
    int start = 0, used = 0;
    for (int base = 0; base < d.tries; base += 32) {
        const int t = base + lane;
        int s = 0;
        bool pass = false;
        if (t < d.tries) {
            s = draw_start(d.u[t], M);
            pass = true;
#pragma unroll
            for (int k = 0; k < kDrawSpeakers; ++k)
                if (k < d.S && pass && (STREAM && W[k] ? draw_silent_stream(*W[k], s, d.len, d.threshold_db)
                                        : I16 && X[k] ? draw_silent_i16(Q[k], X[k], s, d.len, d.threshold_db)
                                                      : draw_silent(Q[k], s, d.len, D[k], d.threshold_db)))
                    pass = false;
        }
        const unsigned ok = __ballot_sync(0xffffffffu, pass);
        if (ok) {
            const int f = __ffs(ok) - 1;
            start = __shfl_sync(0xffffffffu, s, f);
            used = base + f + 1;
            break;
        }
        if (base + 32 >= d.tries) start = __shfl_sync(0xffffffffu, s, d.tries - 1 - base);
    }
    if (lane == 0) {
        *d.start = start;
        if (d.used) *d.used = used;
    }
}

// ----------------------------------------------------------------------------- k_layout
// Layout draws of a plan (ss_layout_draw): one warp per draw.  The warp clears the row's hash map in shared memory,
// then lane 0 draws the row (layout_row, a sequential walk over at most K + 1 selection and 2 * min(K, m) + 2 placement
// draws) and writes the slot's layout arrays.
__global__ void __launch_bounds__(32) k_layout(const LayoutDesc* __restrict__ descs) {
    extern __shared__ int scratch[];
    const LayoutDesc d = descs[blockIdx.x];
    const int cap = d.map_cap;
    for (int i = threadIdx.x; i < cap; i += 32) scratch[i] = -1;
    __syncwarp();
    if (threadIdx.x == 0) layout_row(d, scratch, scratch + cap, scratch + 2 * cap);
}

// Layout draws of a plan with grouped draws (ss_layout_group), launched instead of k_layout: one warp per draw, as
// k_layout, each grouped draw narrowed to its group's utterances (layout_row_grouped; groups[i].group null: k_layout's
// row).  A clamped group sets bit 7.
__global__ void __launch_bounds__(32) k_layout_grouped(const LayoutDesc* __restrict__ descs,
                                                       const LayoutGroup* __restrict__ groups) {
    extern __shared__ int scratch[];
    const LayoutDesc d = descs[blockIdx.x];
    const int cap = d.map_cap;
    for (int i = threadIdx.x; i < cap; i += 32) scratch[i] = -1;
    __syncwarp();
    if (threadIdx.x == 0) {
        const unsigned err = layout_row_grouped(d, groups[blockIdx.x], scratch, scratch + cap, scratch + 2 * cap);
        if (err) atomicOr(&g_dev_err, err);
    }
}

// ----------------------------------------------------------------------------- k_values
// Value draws of a plan (ss_value_draw): one warp per row b, four rows per CTA.  The warp runs the draws in list order,
// its lanes striding over the row's elements (value_row; a distinct row on lane 0, its map in shared memory), with a
// __syncwarp between draws so that a base draw's value is written before a later draw of the row reads it.
constexpr int kValueWarps = 4;
__global__ void __launch_bounds__(32 * kValueWarps) k_values(const ValueDesc* __restrict__ descs, int n, int rows) {
    __shared__ uint32_t map[kValueWarps][2 * kValueMapCap];
    const int w = threadIdx.x >> 5;
    const int b = blockIdx.x * kValueWarps + w;
    if (b >= rows) return;
    for (int r = 0; r < n; ++r) {
        const ValueDesc d = descs[r];
        value_row(d, b, threadIdx.x & 31, 32, map[w], map[w] + kValueMapCap);
        __syncwarp();
    }
}

// ----------------------------------------------------------------------------- k_stage
// Staged slots: at the head of every run (after k_draw, so that drawn starts are final), each pooled slot of a host pool
// and each slot with a dry pick from a host or 16-bit dry pool gets its picked candidate's read set (stage_set) copied
// (from pinned, mapped host memory, or a 16-bit pool's arena) into its staging area, and its view of the candidate
// (StageView), which the head of k_blocks takes.
// A slot of a host pool stages the RIR rows and the dry samples; a slot of a device pool stages only the dry samples of
// its dry pick.  One gridDim.y row of kStageCtas CTAs per slot: every CTA works out the read set (stage_head), then the
// CTAs copy it in 16-byte loads, kStageUnroll of them in flight per thread.
constexpr int kStageCtas = 16, kStageUnroll = 4;
struct StageSlot {
    const PoolEntry* pool;            // the pool's table (a host pool's: x and spec are mapped host addresses)
    const int* pick;
    const int* ws_dev;                // the slot's moving start, or null: ws
    const int* parts;                 // the candidates' K when they differ (pool_parts), else null: K
    const float* gains;               // the pool's gains, or null
    const float* const* dry;          // a host dry pool's signal table (mapped host addresses), or null: no dry pick ...
    const int* dry_pick;              // ... the slot's dry pick ...
    const float* pair;                // ... and its pair gains, or null
    StageView* view;                  // staging area: the view, ...
    float2* spec;                     // ... sets * rows_cap rows (used: sets * rows, back to back) ...
    float* x;                         // ... and the dry samples, whole float4s from xa & ~3 on
    int n, C, K, ws, len;
    int sets;                         // spectra sets staged: 1, 2 with a direct target, 0 for a slot of a device pool
    int n_dry;                        // ... and the dry pool's signal count
    int i16;                          // 1: the dry pool is 16-bit, `dry` holds int16 addresses (k_stage<true> only)
                                      // 2: a stream slot (k_stage<true, TAPS, true> only): `dry` holds its DryStream's
                                      //    address, dry_pick is null
                                      // 3: a bed slot (k_stage<true, TAPS, true, true> only): `dry` holds its
                                      //    BgStream's address, dry_pick is null
};
static_assert(sizeof(StageSlot) == 120, "StageSlot layout");
// k_stage<true, TAPS, true> (a plan with a stream slot) fills such a slot's whole groups [xa & ~3, (xb + 3) & ~3) from
// its layout: the CTA loads the m entries into shared memory, one thread walks them (stream_resolve, bit 5), then
// every thread stores samples of the read set (stream_sample), consecutive threads consecutive samples, so that a
// warp's int16 loads are contiguous within an utterance (coalesced over PCIe from a host arena).
__device__ __forceinline__ void stage_stream_x(const DryStream& d, int x0, int x1, float* __restrict__ xd) {
    __shared__ int s_id[kStreamEntries], s_off[kStreamEntries], s_len[kStreamEntries], s_a[kStreamEntries],
        s_b[kStreamEntries];
    __shared__ const int16_t* s_sig[kStreamEntries];
    __shared__ const int16_t* s_p[kStreamEntries];
    __shared__ int s_k;
    for (int j = threadIdx.x; j < d.m; j += blockDim.x) {
        const int id = d.ids[j];
        const bool ok = id >= 0 && id < d.n;
        s_id[j] = id; s_off[j] = d.offsets[j];
        s_len[j] = ok ? d.lengths[id] : 0;
        s_sig[j] = ok ? d.sig[id] : nullptr;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int k;
        const unsigned err = stream_resolve(s_id, s_off, s_len, s_sig, d.m, d.n, d.cut, s_a, s_b, s_p, &k);
        s_k = k;
        if (err && blockIdx.x == 0) atomicOr(&g_dev_err, err);
    }
    __syncthreads();
    const int nx = x1 - x0, k = s_k, stride = gridDim.x * blockDim.x;
    for (int t0 = blockIdx.x * blockDim.x + threadIdx.x; t0 < nx; t0 += stride * kStageUnroll) {
        float v[kStageUnroll];
#pragma unroll
        for (int u = 0; u < kStageUnroll; ++u) {        // every load issued before the first store
            const int t = t0 + u * stride;
            v[u] = t < nx ? stream_sample(s_a, s_b, s_p, k, x0 + t) : 0.0f;
        }
#pragma unroll
        for (int u = 0; u < kStageUnroll; ++u) if (t0 + u * stride < nx) xd[t0 + u * stride] = v[u];
    }
}
// k_stage<true, TAPS, true, true> (a plan with a bed slot) fills such a slot's groups as stage_stream_x fills a stream
// slot's, from its resolved bed layout (bg_resolve, bit 5; bg_sample): int16 clips through i16_sample, float32 clips as
// they are, whichever the slot's dry pool holds.
__device__ __forceinline__ void stage_bg_x(const BgStream& d, int x0, int x1, float* __restrict__ xd) {
    __shared__ int s_id[kStreamEntries], s_off[kStreamEntries], s_hd[kStreamEntries], s_cnt[kStreamEntries],
        s_len[kStreamEntries], s_a[kStreamEntries], s_b[kStreamEntries];
    __shared__ const char* s_sig[kStreamEntries];
    __shared__ const char* s_p[kStreamEntries];
    __shared__ int s_k;
    for (int j = threadIdx.x; j < d.m; j += blockDim.x) {
        const int id = d.ids[j];
        const bool ok = id >= 0 && id < d.n;
        s_id[j] = id; s_off[j] = d.offsets[j]; s_hd[j] = d.heads[j]; s_cnt[j] = d.counts[j];
        s_len[j] = ok ? d.lengths[id] : 0;
        s_sig[j] = ok ? d.sig[id] : nullptr;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        int k;
        const unsigned err = bg_resolve(s_id, s_off, s_hd, s_cnt, s_len, s_sig, d.i16 ? 2 : 4, d.m, d.n, d.cut, s_a, s_b,
                                        s_p, &k);
        s_k = k;
        if (err && blockIdx.x == 0) atomicOr(&g_dev_err, err);
    }
    __syncthreads();
    const int nx = x1 - x0, k = s_k, stride = gridDim.x * blockDim.x;
    const bool i16 = d.i16 != 0;
    for (int t0 = blockIdx.x * blockDim.x + threadIdx.x; t0 < nx; t0 += stride * kStageUnroll) {
        float v[kStageUnroll];
#pragma unroll
        for (int u = 0; u < kStageUnroll; ++u) {        // every load issued before the first store
            const int t = t0 + u * stride;
            v[u] = t < nx ? bg_sample(s_a, s_b, s_p, k, x0 + t, i16) : 0.0f;
        }
#pragma unroll
        for (int u = 0; u < kStageUnroll; ++u) if (t0 + u * stride < nx) xd[t0 + u * stride] = v[u];
    }
}
// k_stage<true> (a plan with a 16-bit dry pick) reads such a slot's dry samples as 4 int16 at a time from the whole
// groups [xa & ~3, (xb + 3) & ~3) of the picked signal (inside its padded arena) and stores their exact float32 values,
// so that the staging area holds what a float pool's slot stages.
// k_stage<I16, true> (a plan with a slot of a tap-form pool) copies such a slot's tap rows [row0, row0 + rows), one
// contiguous span of the candidate's rows, instead of sets * rows spectra rows, and writes the Source over them that the
// plan's transform launch (k_prepare<false>) turns into the spectra the slot's view names: those k_stage<I16> copies.
template <bool I16, bool TAPS = false, bool STREAM = false, bool BG = false>
__global__ void __launch_bounds__(256) k_stage(const StageSlot* __restrict__ slots, const StageTap* __restrict__ taps) {
    const StageSlot& g = slots[blockIdx.y];
    const StageTap* const tp = TAPS && taps[blockIdx.y].taps ? &taps[blockIdx.y] : nullptr;
    const DryStream* const ds = STREAM && g.i16 == 2 ? reinterpret_cast<const DryStream*>(g.dry) : nullptr;
    const BgStream* const bs = BG && g.i16 == 3 ? reinterpret_cast<const BgStream*>(g.dry) : nullptr;
    const void* const laid = BG && bs ? (const void*)bs : (const void*)ds;   // a stream or bed slot: no dry pick
    __shared__ StageView s_v;
    __shared__ const float* s_src;                      // the signal the dry samples come from
    __shared__ int s_x[2];                              // dry samples copied: whole float4s [s_x[0], s_x[1])
    if (threadIdx.x == 0) {
        const unsigned err = stage_head(g.pool, g.n, *g.pick, g.parts, g.K, g.gains, g.ws_dev, g.ws, g.len, g.C,
                                        g.sets != 0, laid ? nullptr : g.dry, !laid && g.dry ? *g.dry_pick : 0, g.n_dry, s_v,
                                        s_src, s_x[0], s_x[1], g.pair);
        if (err && blockIdx.x == 0) atomicOr(&g_dev_err, err);
    }
    __syncthreads();
    if (STREAM && ds) stage_stream_x(*ds, s_x[0], s_x[1], g.x);   // (the loop below then copies no dry samples)
    if (BG && bs) stage_bg_x(*bs, s_x[0], s_x[1], g.x);
    const PoolEntry& e = s_v.e;
    const size_t nx4 = (STREAM || BG) && laid ? 0 : (size_t)((s_x[1] - s_x[0]) >> 2);
    const size_t per_set = (size_t)s_v.rows * (kSpec / 2);          // float4s per set
    const size_t rows_h = (size_t)e.P * g.C * s_v.K;                 // rows per set of the bank
    const size_t total = nx4 + (TAPS && tp ? (size_t)s_v.rows * (kB / 4) : (size_t)g.sets * per_set);
    const float4* const xs = reinterpret_cast<const float4*>(s_src + s_x[0]);
    const short4* const xs16 = I16 && g.i16 ? reinterpret_cast<const short4*>(reinterpret_cast<const int16_t*>(s_src) + s_x[0])
                                            : nullptr;
    float4* const xd = reinterpret_cast<float4*>(g.x);
    const size_t stride = (size_t)gridDim.x * blockDim.x;
    for (size_t q0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x; q0 < total; q0 += stride * kStageUnroll) {
        float4 v[kStageUnroll];
        float4* dst[kStageUnroll];
#pragma unroll
        for (int u = 0; u < kStageUnroll; ++u) {        // every load issued before the first store
            const size_t q = q0 + u * stride;
            dst[u] = nullptr;
            if (q >= total) continue;
            if (q < nx4) { v[u] = I16 && xs16 ? i16x4_samples(xs16[q]) : xs[q]; dst[u] = xd + q; continue; }
            if (TAPS && tp) {
                const size_t j = q - nx4;
                v[u] = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(e.spec) + (size_t)s_v.row0 * kB)[j];
                dst[u] = reinterpret_cast<float4*>(tp->taps) + j;
                continue;
            }
            const size_t j = q - nx4, set = j / per_set;
            v[u] = reinterpret_cast<const float4*>(e.spec + (set * rows_h + s_v.row0) * kSpec)[j - set * per_set];
            dst[u] = reinterpret_cast<float4*>(g.spec) + j;
        }
#pragma unroll
        for (int u = 0; u < kStageUnroll; ++u) if (dst[u]) *dst[u] = v[u];
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        StageView w = s_v;
        w.e.x = g.x - s_x[0];                           // biased: sample n at x[n] (Source::x)
        if (g.sets) w.e.spec = g.spec;                  // (a device pool's slot keeps its bank's spectra)
        *g.view = w;
        if (TAPS && tp)
            *tp->src = tap_source(tp->taps, g.spec, g.sets > 1 ? e.cut : nullptr, e.P, g.C, s_v.K, s_v.row0, s_v.rows,
                                  tp->zero);
    }
}

// ----------------------------------------------------------------------------- k_loud_crop
// The crops of a plan's loudness slots, after their whole stems were measured: one gridDim.y row per slot, the crop
// and the direct-path crop cut out of the whole stems at the slot's start and scaled by the gain of the run
// (loud_crop_head), float4 at a time when the whole stem, the start, the length and the outputs allow it.
__global__ void __launch_bounds__(256) k_loud_crop(const LoudCrop* __restrict__ crops) {
    const LoudCrop& q = crops[blockIdx.y];
    int start;
    float g;
    const unsigned err = loud_crop_head(q, start, g);
    if (err && blockIdx.x == 0 && threadIdx.x == 0) atomicOr(&g_dev_err, err);
    const long long total = (long long)q.C * q.len, stride = (long long)gridDim.x * blockDim.x;
    const long long i0 = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    for (int dir = 0; dir < 2; ++dir) {
        const float* const src = dir ? q.whole_dir : q.whole;
        float* const dst = dir ? q.out_dir : q.out;
        if (!dst) continue;
        if (((q.N | start | q.len) & 3) == 0 && (((uintptr_t)src | (uintptr_t)dst) & 15) == 0) {
            const long long row4 = q.len >> 2;
            for (long long i = i0; i < total >> 2; i += stride) {
                const long long c = i / row4, t = i - c * row4;
                float4 v = reinterpret_cast<const float4*>(src + c * q.N + start)[t];
                v.x *= g; v.y *= g; v.z *= g; v.w *= g;
                reinterpret_cast<float4*>(dst)[i] = v;
            }
        } else {
            for (long long i = i0; i < total; i += stride) dst[i] = loud_crop_sample(q, start, g, dir, i);
        }
    }
}

extern "C" void ss_plan_destroy(ss_plan* p) {
    if (!p) return;
    cudaSetDevice(p->c->device);
    cudaDeviceSynchronize();
    if (p->exec) cudaGraphExecDestroy(p->exec);
    if (p->s_cap) cudaStreamDestroy(p->s_cap);
    if (p->ev_fork) cudaEventDestroy(p->ev_fork);
    for (int i = 0; i < ss_ctx::kAux; ++i) if (p->ev_join[i]) cudaEventDestroy(p->ev_join[i]);
    if (p->d_desc) cudaFree(p->d_desc);
    for (int i = 0; i < ss_ctx::kAux; ++i) if (p->d_scratch[i]) cudaFree(p->d_scratch[i]);
    delete p;
}

// A plan's mixture with its dereverberation targets (ss_plan_target's direct_out), or null
struct PlanMix : ss_plan_mix { float* dir_out; };

// The descriptor of mixture m of a plan: rows of the callers' `items` outputs (before arrange_chunks regroups them);
// with dir_out, its speakers' direct-path stems and the (S, E) targets
static MixItem mix_describe(const ss_source* items, const PlanMix& m, double* scratch) {
    MixItem d; memset(&d, 0, sizeof(d));
    const ss_source& a = items[m.speakers[0]];
    const int64_t T = a.win_len > 0 ? a.win_len : a.N;
    const bool mono = (m.flags & SS_MIX_MONO) != 0;
    for (int s = 0; s < m.S; ++s) d.spk[s] = items[m.speakers[s]].out;
    for (int q = 0; q < m.M; ++q) d.noise[q] = items[m.noises[q]].out;
    d.sirs = m.sirs; d.snr = m.snr; d.mix = m.mix; d.spk_out = m.speakers_out; d.rms_out = m.rms_db; d.scratch = scratch;
    d.E = mono ? T : (int64_t)a.C * T; d.T = T; d.Cf = mono ? a.C : 1;
    d.S = m.S; d.M = m.M; d.delay = m.noise_delay;
    if (m.dir_out) {
        for (int s = 0; s < m.S; ++s) d.dir[s] = items[m.speakers[s]].out_direct;
        d.dir_out = m.dir_out;
    }
    return d;
}

// The descriptor of draw d of a plan: its readers in the callers' order of `items` (a dry-picked speaker tests its dry
// pool's one-channel tables, D = len; a stream speaker walks its layout through its DryStream, D = len)
static DrawDesc draw_describe(const ss_source* items, const std::vector<PlanSlot>& slots, const ss_plan_draw& d) {
    DrawDesc g; memset(&g, 0, sizeof(g));
    g.start = d.start; g.u = d.u; g.used = d.used; g.tries = d.tries; g.S = d.S; g.threshold_db = d.threshold_db;
    for (int i = 0; i < (int)slots.size(); ++i) {
        const ss_source& it = items[i];
        if (it.win_start_dev != d.start) continue;
        for (int k = 0; k < d.S; ++k) if (d.speakers[k] == i) g.spk[k] = g.n_readers;
        const ss_pool* pl = it.pool;
        g.len = it.win_len;
        DrawReader r = {pl->table, it.pick_dev, pl->level_ptr, pl->n,
                        (double)it.win_len * ((pl->level_flags & SS_MIX_MONO) ? 1 : pl->C), nullptr, nullptr, 0};
        if (const ss_dry_pick* p = slots[i].dry) {
            r.dry_levels = p->pool->level_ptr; r.dry_pick = p->pick_dev; r.n_dry = p->pool->n; r.D = it.win_len;
            r.dry16 = p->pool->i16 ? 1 : 0;
        }
        if (slots[i].ws) { r.dry_pick = reinterpret_cast<const int*>(slots[i].ws); r.dry16 = 2; r.D = it.win_len; }
        g.r[g.n_readers++] = r;
    }
    return g;
}

// Staging area of a pooled slot of a host pool with windows of win_len (stage_cap), worked out once per pool and length
static std::pair<int, int> stage_cap(ss_pool* pl, int win_len) {
    for (const auto& q : pl->stage_caps) if (q.first == win_len) return q.second;
    std::vector<const int*> bounds;
    std::vector<int> N(pl->n), P(pl->n);
    for (int i = 0; i < pl->n; ++i) {
        N[i] = pl->host[i].N; P[i] = pl->host[i].P;
        if (pl->mode == SS_MOVING_BOUNDS) bounds.push_back(pl->bounds_host.data() + pl->bounds_off[i]);
    }
    int rows, nx;
    stage_cap(bounds.empty() ? nullptr : bounds.data(), N.data(), P.data(), pl->parts_host.data(), pl->n, pl->C, win_len,
              rows, nx);
    pl->stage_caps.push_back({win_len, {rows, nx}});
    return {rows, nx};
}
// (spectra sets it stages: direct_sets for a slot of a host pool, 0 for a slot of a device pool, which stages dry samples only)
static int stage_sets(const ss_source& it) { return it.pool->host_res ? direct_sets(it) : 0; }
// A slot's staging area (stage_area): view | spectra | dry samples | (a slot of a tap-form pool) tap rows
static StageArea stage_area_of(const ss_source& it) {
    const std::pair<int, int> cap = stage_cap(const_cast<ss_pool*>(it.pool), it.win_len);
    return stage_area(stage_sets(it), cap.first, cap.second, it.pool->taps);
}

// K of a layout draw (ss_layout_draw): the most a row can select.  A stream: the largest k whose k shortest utterances
// fit in `total` (at least 1).  A bed: the most clips whose selection lengths stay below 0.4 * total, plus the one that
// crosses it (at most n).
static int64_t layout_bound(const ss_layout_draw& L, const ss_dry_pool* dp, bool bed,
                            const ss_layout_group* grp = nullptr) {
    if (grp) {                                          // a grouped stream: the largest K of its groups
        int64_t K = 1;
        for (int g = 0; g < grp->n_groups; ++g) {
            std::vector<int64_t> v(dp->N.begin() + grp->bounds[g], dp->N.begin() + grp->bounds[g + 1]);
            std::sort(v.begin(), v.end());
            int64_t acc = 0, k = 0;
            for (int64_t l : v) {
                if (acc + l > L.total) break;
                acc += l; ++k;
            }
            K = std::max(K, k);
        }
        return K;
    }
    std::vector<int64_t> v(dp->N.begin(), dp->N.end());
    if (L.select_lengths) v.assign(L.select_lengths, L.select_lengths + dp->n);
    std::sort(v.begin(), v.end());
    int64_t acc = 0, k = 0;
    for (int64_t l : v) {
        if (bed ? !((double)(acc + l) < 0.4 * (double)L.total) : acc + l > L.total) break;
        acc += l; ++k;
    }
    return bed ? std::min<int64_t>(dp->n, k + 1) : std::max<int64_t>(1, k);
}

// Lay out, fill and upload a plan's descriptors.  The host fills one image, each section at a 256-byte boundary: the
// chunk descriptors, the mixtures' MixItems, the draws' DrawDescs, the staged slots' StageSlots, the tap block
// (tap_block, with slots of tap-form pools), the streams' DryStreams and the beds' BgStreams (caller order) and the
// clip lengths of each dry pool the streams and beds use, the layout draws' LayoutDescs and their select lengths, the
// value draws' ValueDescs, and for loudness slots their LoudItems, work-item offsets, LoudCrops and gating tables; one
// copy uploads it.  Behind the image, written by the device only and never uploaded:
// one scratch block per mixture, the staged slots' staging areas, then per loudness slot its whole stems, its loudness
// scratch and (without a result_dev) its result.  slots[i] is caller item i's record; plan_build notes where its view,
// its DryStream and its BgStream landed.  A loudness slot is chunked, staged and rendered as the window [0, N) into its
// whole stems; draws and mixtures keep reading the caller's item, whose crop k_loud_crop writes.
static int plan_build(ss_plan* p, const ss_source* caller_items, const Shape* caller_shapes,
                      std::vector<PlanSlot>& slots, const std::vector<PlanMix>& mix, const ss_plan_draw* draws,
                      int n_draws, const ss_layout_draw* layouts, int n_layouts, const ss_value_draw* values,
                      int n_values, const ss_layout_group* groups, int n_grouped) {
    ss_ctx* c = p->c;
    const int n_items = (int)slots.size();
    std::vector<int> cuts, order;
    std::vector<ss_source> arranged;
    std::vector<Shape> arranged_shapes;
    std::vector<ss_source> rendered(caller_items, caller_items + n_items);   // loudness slots: the window [0, N)
    std::vector<Shape> rendered_shapes(caller_shapes, caller_shapes + n_items);
    std::vector<int> loud;                               // the loudness slots, in caller order
    for (int i = 0; i < n_items; ++i) {
        if (!slots[i].lufs && !slots[i].traj) continue;
        ss_source& w = rendered[i];
        if (slots[i].lufs) {
            w.win_start = 0; w.win_start_dev = nullptr; w.win_len = w.pool->host[0].N;
            loud.push_back(i);
        }
        rendered_shapes[i] = shape_pooled(w, slots[i].traj != nullptr);
    }
    arrange_chunks(c, rendered.data(), rendered_shapes.data(), n_items, arranged, arranged_shapes, cuts, &order);
    const ss_source* items = arranged.data(); const Shape* shapes = arranged_shapes.data();
    std::vector<PlanSlot*> rec(arranged.size());         // rec[i]: the record of arranged item i
    std::vector<int> staged;    // arranged items that are slots of host pools, host or 16-bit dry picks, stream and bed
    int n_tap = 0, n_strm = 0, n_bg = 0;                 // slots
    for (int i = 0; i < (int)arranged.size(); ++i) {
        rec[i] = &slots[order[i]];
        const PlanSlot& r = *rec[i];
        n_strm += r.strm ? 1 : 0;
        n_bg += r.bg ? 1 : 0;
        if (items[i].pool && (items[i].pool->host_res || (r.dry && r.dry->pool->padded()) || r.strm || r.bg)) {
            staged.push_back(i);
            n_tap += items[i].pool->taps ? 1 : 0;
        }
    }
    if (staged.size() > 65535) return SS_ERR_UNSUPPORTED;   // one gridDim.y row of k_stage per slot
    size_t at = 0;
    auto take = [&at](size_t bytes) { const size_t o = at; at = align_up(at + bytes, 256); return o; };
    const size_t n_chunks = cuts.size() - 1;
    std::vector<size_t> off(n_chunks);
    size_t scratch_need[ss_ctx::kAux] = {};
    for (size_t k = 0; k < n_chunks; ++k) {
        off[k] = take(chunk_desc_bytes(items, shapes, cuts[k], cuts[k + 1]));
        const size_t sb = chunk_scratch_bytes(items, shapes, cuts[k], cuts[k + 1]);
        size_t& m = scratch_need[n_chunks < 2 ? 0 : k % ss_ctx::kAux];
        m = sb > m ? sb : m;
    }
    const size_t mix_off = take(sizeof(MixItem) * mix.size());
    const size_t draw_off = take(sizeof(DrawDesc) * n_draws);
    const size_t stage_off = take(sizeof(StageSlot) * staged.size());
    const TapBlock tb = tap_block(at, (int)staged.size(), n_tap);
    if (n_tap) at = tb.end;
    const size_t wdesc_off = take(sizeof(DryStream) * n_strm);
    const size_t bdesc_off = take(sizeof(BgStream) * n_bg);
    std::vector<const ss_dry_pool*> wpools;              // each with its lengths at wlen_off
    std::vector<size_t> wlen_off;
    for (const PlanSlot& s : slots)
        if (s.clips() && std::find(wpools.begin(), wpools.end(), s.clips()) == wpools.end()) {
            wpools.push_back(s.clips());
            wlen_off.push_back(take(sizeof(int32_t) * (size_t)s.clips()->n));
        }
    auto lengths_at = [&](const ss_dry_pool* dp) {
        return wlen_off[std::find(wpools.begin(), wpools.end(), dp) - wpools.begin()];
    };
    const size_t ldesc_off = take(sizeof(LayoutDesc) * n_layouts);
    std::vector<size_t> lsel_off(n_layouts);             // a bed draw's select_lengths
    for (int k = 0; k < n_layouts; ++k)
        if (layouts[k].select_lengths) lsel_off[k] = take(sizeof(int32_t) * (size_t)slots[layouts[k].slot].clips()->n);
    const size_t lgrp_off = n_grouped ? take(sizeof(LayoutGroup) * n_layouts) : 0;   // with grouped draws: one each
    std::vector<size_t> gb_off(n_grouped);                // a grouped draw's bounds
    for (int j = 0; j < n_grouped; ++j) gb_off[j] = take(sizeof(int32_t) * ((size_t)groups[j].n_groups + 1));
    const size_t vdesc_off = take(sizeof(ValueDesc) * n_values);
    const int n_loud = (int)loud.size();
    std::vector<ss_post_lufs> gating(n_loud);
    for (int k = 0; k < n_loud; ++k) gating[k] = slots[loud[k]].lufs->gating;
    const GatingTables gtabs = gating_tables(gating.data(), n_loud);
    const size_t loud_off = take(sizeof(LoudItem) * n_loud);
    const size_t lpre_off = take(sizeof(int) * (n_loud + 1));
    const size_t crop_off = take(sizeof(LoudCrop) * n_loud);
    const size_t gtab_off = take(gtabs.bytes.size());
    const size_t image = at;
    const size_t scr_bytes = sizeof(double) * (size_t)ss_mix_scratch_doubles();
    const size_t scr_off = take(scr_bytes * mix.size());
    std::vector<size_t> area_off(staged.size());
    for (size_t k = 0; k < staged.size(); ++k) area_off[k] = take(stage_area_of(items[staged[k]]).end);
    // a loudness slot's whole stem (C * N floats), its whole direct-path stem, loudness scratch and result
    std::vector<size_t> whole_off(n_items), wdir_off(n_items), lscr_off(n_loud), lres_off(n_loud);
    for (int k = 0; k < n_loud; ++k) {
        const ss_source& w = rendered[loud[k]];
        const size_t stem = sizeof(float) * (size_t)w.C * w.win_len;
        whole_off[loud[k]] = take(stem);
        if (w.flags & SS_DIRECT_TARGET) wdir_off[loud[k]] = take(stem);
        lscr_off[k] = take(loud_scratch_bytes(gating[k], w.C));
        if (!slots[loud[k]].lufs->result_dev) lres_off[k] = take(2 * sizeof(double));
    }
    CK(cudaEventCreateWithFlags(&p->ev_fork, cudaEventDisableTiming));
    for (int i = 0; i < ss_ctx::kAux; ++i) CK(cudaEventCreateWithFlags(&p->ev_join[i], cudaEventDisableTiming));
    CK(cudaStreamCreateWithFlags(&p->s_cap, cudaStreamNonBlocking));
    CK(cudaMalloc((void**)&p->d_desc, at + 256));
    for (int i = 0; i < ss_ctx::kAux; ++i)
        if (scratch_need[i]) CK(cudaMalloc((void**)&p->d_scratch[i], align_up(scratch_need[i], 1 << 20)));
    char* const d = p->d_desc;
    std::vector<char> host(image, 0);
    for (size_t i = 0; i < arranged.size(); ++i) {       // loudness slots render into their whole stems
        if (!rec[i]->lufs) continue;
        arranged[i].out = (float*)(d + whole_off[order[i]]);
        if (arranged[i].flags & SS_DIRECT_TARGET) arranged[i].out_direct = (float*)(d + wdir_off[order[i]]);
    }
    if (n_loud) {
        if (!gtabs.bytes.empty()) memcpy(host.data() + gtab_off, gtabs.bytes.data(), gtabs.bytes.size());
        int* const prefix = (int*)(host.data() + lpre_off);
        int total = 0;
        for (int k = 0; k < n_loud; ++k) {
            const int i = loud[k];
            const ss_stream_lufs& q = *slots[i].lufs;
            const ss_source& w = rendered[i];
            const ss_source& a = caller_items[i];
            double* const result = q.result_dev ? q.result_dev : (double*)(d + lres_off[k]);
            const float* const whole = (const float*)(d + whole_off[i]);
            const float* const wdir = (w.flags & SS_DIRECT_TARGET) ? (const float*)(d + wdir_off[i]) : nullptr;
            LoudItem it = to_item(loud_item(q.gating, d + gtab_off + gtabs.at[k], whole, nullptr, w.win_len, w.C,
                                            (double*)(d + lscr_off[k]), result));
            it.target_dev = q.target_dev;
            memcpy(host.data() + loud_off + sizeof(LoudItem) * k, &it, sizeof(it));
            const LoudCrop crop = {whole, wdir, a.out, wdir ? a.out_direct : nullptr, a.win_start_dev, q.target_dev,
                                   result, a.win_start, a.win_len, w.win_len, w.C};
            memcpy(host.data() + crop_off + sizeof(LoudCrop) * k, &crop, sizeof(crop));
            prefix[k] = total;
            total += w.C * q.gating.n_e;
            p->crop_ctas = std::max(p->crop_ctas, (int)std::min<long long>(64, ((long long)w.C * a.win_len + 1023) / 1024));
        }
        prefix[n_loud] = total;
        p->d_loud = (const LoudItem*)(d + loud_off);
        p->d_loud_prefix = (const int*)(d + lpre_off);
        p->d_crop = (const LoudCrop*)(d + crop_off);
        p->n_loud = n_loud; p->loud_total = total; p->loud_rate = gating[0].rate;
    }
    for (int i = 0, k = 0, kb = 0; i < n_items; ++i) {   // the streams and beds first: staged slots and draws name them
        const ss_dry_pool* dp = slots[i].clips();
        if (!dp) continue;
        const int* const lengths = (const int*)(d + lengths_at(dp));
        int cut = 0;
        for (const PoolEntry& e : caller_items[i].pool->host) cut = std::max(cut, e.N);
        if (const ss_dry_stream* w = slots[i].strm) {
            ((DryStream*)(host.data() + wdesc_off))[k] = {w->ids_dev, w->offsets_dev, lengths,
                                                          (const int16_t* const*)dp->ptrs,
                                                          dp->levels ? dp->level_ptr : nullptr, w->m, dp->n, cut, 0};
            slots[i].ws = (const DryStream*)(d + wdesc_off) + k++;
        } else {
            const ss_bg_stream& b = *slots[i].bg;
            ((BgStream*)(host.data() + bdesc_off))[kb] = {b.ids_dev, b.offsets_dev, b.heads_dev, b.counts_dev, lengths,
                                                          (const char* const*)dp->ptrs, b.m, dp->n, cut, dp->i16 ? 1 : 0};
            slots[i].wb = (const BgStream*)(d + bdesc_off) + kb++;
        }
    }
    for (size_t j = 0; j < wpools.size(); ++j)
        memcpy(host.data() + wlen_off[j], wpools[j]->N.data(), sizeof(int32_t) * (size_t)wpools[j]->n);
    for (int k = 0; k < n_layouts; ++k) {                // the layout draws write their slots' own layout arrays
        const ss_layout_draw& L = layouts[k];
        const PlanSlot& r = slots[L.slot];
        const ss_dry_pool* dp = r.clips();
        LayoutDesc& g = ((LayoutDesc*)(host.data() + ldesc_off))[k];
        g.rng = L.rng_dev; g.lengths = (const int*)(d + lengths_at(dp));
        if (L.select_lengths) {
            memcpy(host.data() + lsel_off[k], L.select_lengths, sizeof(int32_t) * (size_t)dp->n);
            g.select = (const int*)(d + lsel_off[k]);
        }
        if (r.strm) {
            g.ids = const_cast<int*>(r.strm->ids_dev); g.offsets = const_cast<int*>(r.strm->offsets_dev); g.m = r.strm->m;
        } else {
            g.ids = const_cast<int*>(r.bg->ids_dev); g.offsets = const_cast<int*>(r.bg->offsets_dev);
            g.heads = const_cast<int*>(r.bg->heads_dev); g.counts = const_cast<int*>(r.bg->counts_dev); g.m = r.bg->m;
        }
        g.n = dp->n; g.total = L.total; g.gap_max = 10 * L.sample_rate; g.r = k;
        g.K = (int)layout_bound(L, dp, r.bg != nullptr, r.group);
        g.map_cap = layout_map_cap(g.K);
        p->layout_smem = std::max(p->layout_smem, (int)sizeof(int) * layout_scratch_ints(g.K));
    }
    for (int j = 0; j < n_grouped; ++j) {                // grouped draws: their group and bounds (others: null)
        const ss_layout_group& q = groups[j];
        memcpy(host.data() + gb_off[j], q.bounds, sizeof(int32_t) * ((size_t)q.n_groups + 1));
        LayoutGroup& e = ((LayoutGroup*)(host.data() + lgrp_off))[q.layout];
        e.group = q.group_dev; e.bounds = (const int*)(d + gb_off[j]); e.G = q.n_groups;
    }
    for (int k = 0; k < n_values; ++k) {                 // the value draws write the caller's per-run inputs
        const ss_value_draw& v = values[k];
        ValueDesc& g = ((ValueDesc*)(host.data() + vdesc_off))[k];
        g.out = v.out; g.rng = v.rng_dev;
        g.base = v.base >= 0 ? (const int*)values[v.base].out : nullptr;
        g.low = v.low; g.high = v.high; g.ilow = v.ilow; g.n = (uint32_t)((int64_t)v.ihigh - v.ilow);
        g.kind = v.kind; g.k = v.k; g.r = k; g.stride = v.base >= 0 ? v.stride : 0;
    }
    for (size_t k = 0; k < staged.size(); ++k) {
        const ss_source& it = items[staged[k]];
        PlanSlot& r = *rec[staged[k]];
        const ss_pool* pl = it.pool;
        StageSlot& g = ((StageSlot*)(host.data() + stage_off))[k];
        g.pool = pl->table; g.pick = it.pick_dev; g.ws_dev = it.win_start_dev; g.parts = pl->parts; g.gains = pl->gains;
        g.n = pl->n; g.C = pl->C; g.K = pl->K; g.ws = it.win_start; g.len = it.win_len; g.sets = stage_sets(it);
        if (const ss_dry_pick* dp = r.dry) {
            g.dry = dp->pool->ptrs; g.dry_pick = dp->pick_dev; g.n_dry = dp->pool->n; g.pair = r.pair;
            g.i16 = dp->pool->i16 ? 1 : 0;
            p->stage16 = p->stage16 || dp->pool->i16;
        }
        if (r.ws) {                                     // (k_stage reads the layout through its DryStream)
            g.dry = reinterpret_cast<const float* const*>(r.ws); g.n_dry = r.strm->pool->n; g.i16 = 2;
            p->stage_stream = true;
        }
        if (r.wb) {                                     // (k_stage reads the layout through its BgStream)
            g.dry = reinterpret_cast<const float* const*>(r.wb); g.n_dry = r.bg->pool->n; g.i16 = 3;
            p->stage_bg = true;
        }
        const std::pair<int, int> cap = stage_cap(const_cast<ss_pool*>(pl), it.win_len);
        const StageArea sa = stage_area_of(it);
        char* const a = d + area_off[k];
        g.view = (StageView*)(a + sa.view);
        g.spec = g.sets ? (float2*)(a + sa.spec) : nullptr;
        g.x = (float*)(a + sa.x);
        r.view = g.view;
        if (pl->taps) {                                 // its tap rows, transform Source and CTA range
            const int t = p->n_tap++;
            StageTap& q = ((StageTap*)(host.data() + tb.taps))[k];
            q.taps = (float*)(a + sa.taps);
            q.src = (Source*)(d + tb.src) + t;
            q.zero = (int*)(d + tb.zero);
            int* const prefix = (int*)(host.data() + tb.prefix);
            prefix[t + 1] = prefix[t] + g.sets * ((cap.first + 1) >> 1);   // pairs of the most rows any run stages
        }
    }
    p->chunks.resize(n_chunks);
    for (size_t k = 0; k < n_chunks; ++k)
        chunk_describe(items, shapes, cuts[k], cuts[k + 1], host.data() + off[k], d + off[k],
                       p->d_scratch[n_chunks < 2 ? 0 : k % ss_ctx::kAux], c->sm_count, &p->chunks[k], rec.data());
    for (size_t k = 0; k < mix.size(); ++k) {
        ((MixItem*)(host.data() + mix_off))[k] =
            mix_describe(caller_items, mix[k], (double*)(d + scr_off + scr_bytes * k));
        p->mix_direct = p->mix_direct || mix[k].dir_out;
    }
    for (int k = 0; k < n_draws; ++k) {
        DrawDesc& g = ((DrawDesc*)(host.data() + draw_off))[k];
        g = draw_describe(caller_items, slots, draws[k]);
        for (int j = 0; j < g.S; ++j) {
            p->draw16 = p->draw16 || g.r[g.spk[j]].dry16;
            p->draw_stream = p->draw_stream || g.r[g.spk[j]].dry16 == 2;
        }
    }
    CK(cudaMemcpy(d, host.data(), image, cudaMemcpyHostToDevice));
    if (!mix.empty()) { p->d_mix = (const MixItem*)(d + mix_off); p->n_mix = (int)mix.size(); }
    if (n_draws > 0) { p->d_draw = (const DrawDesc*)(d + draw_off); p->n_draw = n_draws; }
    if (n_layouts > 0) { p->d_layout = (const LayoutDesc*)(d + ldesc_off); p->n_layout = n_layouts; }
    if (n_grouped > 0) p->d_layout_group = (const LayoutGroup*)(d + lgrp_off);
    if (n_values > 0) {
        p->d_value = (const ValueDesc*)(d + vdesc_off); p->n_value = n_values; p->value_rows = values[0].rows;
    }
    if (!staged.empty()) { p->d_stage = (const StageSlot*)(d + stage_off); p->n_stage = (int)staged.size(); }
    if (n_tap) {
        p->tap_ctas = ((const int*)(host.data() + tb.prefix))[n_tap];
        p->d_taps = (const StageTap*)(d + tb.taps);
        p->d_tap_src = (const Source*)(d + tb.src);
        p->d_tap_prefix = (const int*)(d + tb.prefix);
    }
    return SS_OK;
}

// Byte ranges of a plan's mixtures: every range a mixture writes (mix, speakers_out, rms_db) meets no other range of
// the plan - no other written range, no mixture's sirs / snr, nothing an item reads or writes.  One sort and one sweep.
// `input`: a small per-run input that a value draw may write (validate_value_ranges).
struct ByteRange { uintptr_t lo, hi; bool written, input; };
static void add_range(std::vector<ByteRange>& r, const void* p, uint64_t bytes, bool written, bool input = false) {
    if (p && bytes > 0) r.push_back({(uintptr_t)p, (uintptr_t)p + (uintptr_t)bytes, written, input});
}
static bool written_ranges_disjoint(std::vector<ByteRange>& r) {
    std::sort(r.begin(), r.end(), [](const ByteRange& a, const ByteRange& b) { return a.lo < b.lo; });
    uintptr_t end_any = 0, end_written = 0;                 // furthest end of the ranges that start before this one
    for (const ByteRange& x : r) {
        if (x.lo < (x.written ? end_any : end_written)) return false;
        end_any = x.hi > end_any ? x.hi : end_any;
        if (x.written) end_written = x.hi > end_written ? x.hi : end_written;
    }
    return true;
}

// A plan's start draws (include/sonicsim_b200.h, ss_plan_draw), all but the byte ranges (validate_mixes)
static int validate_draws(const ss_source* items, const std::vector<PlanSlot>& slots, const ss_plan_draw* draws,
                          int n_draws) {
    const int n_items = (int)slots.size();
    if (n_draws > kMaxDraws) return SS_ERR_UNSUPPORTED;
    for (int k = 0; k < n_draws; ++k) {
        const ss_plan_draw& d = draws[k];
        if (d.S > kDrawSpeakers || d.tries > kDrawTries) return SS_ERR_UNSUPPORTED;
        if (d.S < 1 || d.tries < 1 || !d.start || !d.u || !isfinite(d.threshold_db)) return SS_ERR_INVALID;
        if (((uintptr_t)d.u & 7) || ((uintptr_t)d.used & 3)) return SS_ERR_INVALID;
        for (int j = 0; j < k; ++j) if (draws[j].start == d.start) return SS_ERR_INVALID;
        for (int s = 0; s < d.S; ++s) {
            const int i = d.speakers[s];
            if (i < 0 || i >= n_items) return SS_ERR_INVALID;
            for (int j = 0; j < s; ++j) if (d.speakers[j] == i) return SS_ERR_INVALID;
            const ss_source& it = items[i];
            // level tables to test: the dry pool's for a dry-picked speaker, else the pool's
            if (!it.pool || it.win_start_dev != d.start) return SS_ERR_INVALID;
            const PlanSlot& r = slots[i];
            if (r.strm ? !r.strm->pool->levels : r.dry ? !r.dry->pool->levels : !it.pool->levels) return SS_ERR_INVALID;
        }
        int readers = 0, len = -1;
        for (int i = 0; i < n_items; ++i) {
            const ss_source& it = items[i];
            if (it.win_start_dev != d.start) continue;
            if (!it.pool || (len >= 0 && it.win_len != len)) return SS_ERR_INVALID;
            len = it.win_len;
            ++readers;
        }
        if (readers > kDrawReaders) return SS_ERR_UNSUPPORTED;
    }
    return SS_OK;
}

// (a mixture's dir_out, when not null: S * E floats written, and every speaker of the mixture needs a direct-path stem)
// `ranges` receives every range the plan reads or writes (validate_value_ranges).
static int validate_mixes(const ss_source* items, const std::vector<PlanSlot>& slots, const std::vector<PlanMix>& mix,
                          const ss_plan_draw* draws, int n_draws, std::vector<ByteRange>& ranges) {
    const int n_items = (int)slots.size();
    if (mix.size() > 65535) return SS_ERR_UNSUPPORTED;      // one gridDim.y row per mixture
    std::vector<ByteRange> r;
    // a draw writes its start (which only its readers read) and `used`, and reads its u
    for (int k = 0; k < n_draws; ++k) {
        add_range(r, draws[k].start, 4, true);
        add_range(r, draws[k].used, 4, true);
        add_range(r, draws[k].u, 8 * (uint64_t)draws[k].tries, false, true);
    }
    for (const PlanMix& m : mix) {
        if (m.S < 1 || m.M < 1 || m.S > kMixStems || m.M > kMixStems) return SS_ERR_UNSUPPORTED;
        if (!m.snr || (m.S > 1 && !m.sirs) || !m.mix || (m.flags & ~SS_MIX_MONO) || m.noise_delay < 0)
            return SS_ERR_INVALID;
        int stems[2 * kMixStems];
        for (int s = 0; s < m.S; ++s) stems[s] = m.speakers[s];
        for (int q = 0; q < m.M; ++q) stems[m.S + q] = m.noises[q];
        for (int j = 0; j < m.S + m.M; ++j) {
            if (stems[j] < 0 || stems[j] >= n_items) return SS_ERR_INVALID;
            for (int i = 0; i < j; ++i) if (stems[i] == stems[j]) return SS_ERR_INVALID;
        }
        const ss_source& a = items[stems[0]];
        const int64_t T = a.win_len > 0 ? a.win_len : a.N;
        for (int j = 1; j < m.S + m.M; ++j) {
            const ss_source& b = items[stems[j]];
            if (b.C != a.C || (b.win_len > 0 ? b.win_len : b.N) != T) return SS_ERR_INVALID;
        }
        if (m.dir_out)
            for (int s = 0; s < m.S; ++s) if (!(items[m.speakers[s]].flags & SS_DIRECT_TARGET)) return SS_ERR_INVALID;
        const uint64_t E = (m.flags & SS_MIX_MONO) ? (uint64_t)T : (uint64_t)a.C * T;
        add_range(r, m.mix, 4 * E, true);
        add_range(r, m.dir_out, 4 * E * m.S, true);
        add_range(r, m.speakers_out, 4 * E * m.S, true);
        add_range(r, m.rms_db, 4 * (uint64_t)m.S, true);
        add_range(r, m.sirs, 4 * (uint64_t)(m.S - 1), false, true);
        add_range(r, m.snr, 4, false, true);
    }
    for (int i = 0; i < n_items; ++i) {
        const ss_source& it = items[i];
        const uint64_t n_out = 4 * (uint64_t)it.C * (it.win_len > 0 ? it.win_len : it.N);
        add_range(r, it.x, 4 * (uint64_t)it.N, false);
        add_range(r, it.rir, 4 * (uint64_t)it.P * it.C * it.L, false);
        add_range(r, it.out, n_out, false);
        if (it.flags & SS_DIRECT_TARGET) add_range(r, it.out_direct, n_out, false);
        if (it.mode == SS_MOVING_BOUNDS) add_range(r, it.bounds, 4 * (uint64_t)it.P, false);
        if (it.mode == SS_MOVING_INDEXED) {
            add_range(r, it.idx, 4 * (uint64_t)it.N, false);
            add_range(r, it.w, 4 * (uint64_t)it.N, false);
        }
        bool drawn = false;
        for (int k = 0; k < n_draws; ++k) drawn = drawn || draws[k].start == it.win_start_dev;
        if (!drawn) add_range(r, it.win_start_dev, 4, false, true);
        add_range(r, it.pick_dev, 4, false, true);
    }
    // a pooled slot may read any candidate: every candidate's x and bounds, once per pool
    std::vector<const ss_pool*> pools;
    for (int i = 0; i < n_items; ++i)
        if (items[i].pool && std::find(pools.begin(), pools.end(), items[i].pool) == pools.end()) pools.push_back(items[i].pool);
    for (const ss_pool* pl : pools)
        for (const PoolEntry& e : pl->host) {
            add_range(r, e.x, 4 * (uint64_t)e.N, false);
            add_range(r, e.bounds, 4 * (uint64_t)e.P, false);
        }
    // a dry-picked slot may read any signal of its dry pool, and reads its dry pick; a stream slot reads its layout; a
    // bed slot reads its layout and may read any clip of its dry pool; a drawn slot writes its layout and reads its rng
    std::vector<const ss_dry_pool*> dpools;
    for (const PlanSlot& s : slots) {
        if (s.dry) {
            add_range(r, s.dry->pick_dev, 4, false, true);
            if (std::find(dpools.begin(), dpools.end(), s.dry->pool) == dpools.end()) dpools.push_back(s.dry->pool);
        }
        const bool drawn = s.layout != nullptr;
        if (drawn) add_range(r, s.layout->rng_dev, 16, false);
        if (s.group) add_range(r, s.group->group_dev, 4, false, true);   // (a value draw may write it)
        if (s.strm) {
            add_range(r, s.strm->ids_dev, 4 * (uint64_t)s.strm->m, drawn);
            add_range(r, s.strm->offsets_dev, 4 * (uint64_t)s.strm->m, drawn);
        }
        if (s.bg) {                                         // a bed slot reads its layout and any clip of its pool
            for (const int32_t* a : {s.bg->ids_dev, s.bg->offsets_dev, s.bg->heads_dev, s.bg->counts_dev})
                add_range(r, a, 4 * (uint64_t)s.bg->m, drawn);
            if (std::find(dpools.begin(), dpools.end(), s.bg->pool) == dpools.end()) dpools.push_back(s.bg->pool);
        }
        if (s.lufs) {                                       // a loudness slot reads its target, writes its result
            add_range(r, s.lufs->target_dev, 8, false, true);
            add_range(r, s.lufs->result_dev, 16, true);
        }
        if (s.traj) {                                       // a trajectory meets nothing else the plan reads or writes
            add_range(r, s.traj->path_dev, 12, true);
            add_range(r, s.traj->bounds_dev, 4 * (uint64_t)items[s.traj->slot].pool->p_max, true);
        }
    }
    for (const ss_dry_pool* dp : dpools)                    // (a host or 16-bit dry pool owns its arena: nothing a plan writes)
        if (!dp->padded())
            for (int i = 0; i < dp->n; ++i) add_range(r, dp->x[i], 4 * (uint64_t)dp->N[i], false);
    // the items' outputs count as read above (mixtures read them); a layout draw's rng and group meet none of them
    // either
    for (const PlanSlot& s : slots) {
        if (!s.layout) continue;
        for (int q = 0; q < (s.group ? 2 : 1); ++q) {
            const uintptr_t lo = q ? (uintptr_t)s.group->group_dev : (uintptr_t)s.layout->rng_dev, hi = lo + (q ? 4 : 16);
            for (int i = 0; i < n_items; ++i) {
                const ss_source& it = items[i];
                const uint64_t n_out = 4 * (uint64_t)it.C * (it.win_len > 0 ? it.win_len : it.N);
                for (const float* o : {it.out, (it.flags & SS_DIRECT_TARGET) ? it.out_direct : nullptr})
                    if (o && (uintptr_t)o < hi && lo < (uintptr_t)o + n_out) return SS_ERR_INVALID;
            }
        }
    }
    if (!written_ranges_disjoint(r)) return SS_ERR_INVALID;
    ranges = std::move(r);
    return SS_OK;
}

// A plan's dry picks (include/sonicsim_b200.h, ss_dry_pick), all but the byte ranges (validate_mixes): the record of
// each pick's slot receives the pick and the device table of its pair gains (pair_gains[k] of pick k), or null
static int validate_dry_picks(const ss_ctx* c, const ss_source* items, const ss_dry_pick* picks,
                              const ss_pair_gains* const* pair_gains, int n_picks, std::vector<PlanSlot>& slots) {
    for (int k = 0; k < n_picks; ++k) {
        const ss_dry_pick& d = picks[k];
        if (d.slot < 0 || d.slot >= (int)slots.size() || slots[d.slot].dry) return SS_ERR_INVALID;   // one per slot
        if (!d.pool || d.pool->c != c || !d.pick_dev || ((uintptr_t)d.pick_dev & 3)) return SS_ERR_INVALID;
        const ss_pool* pl = items[d.slot].pool;
        const ss_pair_gains* const t = pair_gains ? pair_gains[k] : nullptr;
        // a pooled slot whose every candidate's N the dry pool's shortest signal covers, on a pool with gains only with
        // pair gains (the pool's were measured with the candidates' own x) of this pool and dry pool; a slot of a host
        // pool only from a host or 16-bit dry pool, whose arena pads every signal to the whole groups k_stage reads
        if (!pl || (pl->host_res && !d.pool->padded()) || (pl->gains && !t)) return SS_ERR_INVALID;
        if (t && (t->pool != pl || t->dry != d.pool)) return SS_ERR_INVALID;
        for (const PoolEntry& e : pl->host) if (e.N > d.pool->n_min) return SS_ERR_INVALID;
        slots[d.slot].dry = &d;
        slots[d.slot].pair = t ? t->gains : nullptr;
    }
    return SS_OK;
}

// A plan's dry streams (include/sonicsim_b200.h, ss_dry_stream), all but the draws' tables (validate_draws) and the
// byte ranges (validate_mixes): the record of each stream's slot receives the stream
static int validate_streams(const ss_ctx* c, const ss_source* items, const ss_dry_stream* streams, int n_streams,
                            std::vector<PlanSlot>& slots) {
    for (int k = 0; k < n_streams; ++k) {
        const ss_dry_stream& w = streams[k];
        if (w.slot < 0 || w.slot >= (int)slots.size() || slots[w.slot].strm || slots[w.slot].dry) return SS_ERR_INVALID;
        const ss_pool* pl = items[w.slot].pool;
        // a pooled slot of a pool without loudness gains (a stream has no fixed pair to measure), over a 16-bit dry
        // pool of this context, with a layout of 1..kStreamEntries aligned device entries
        if (!pl || pl->gains || !w.pool || w.pool->c != c || !w.pool->i16) return SS_ERR_INVALID;
        if (w.m < 1 || w.m > kStreamEntries || !w.ids_dev || !w.offsets_dev || ((uintptr_t)w.ids_dev & 3) ||
            ((uintptr_t)w.offsets_dev & 3))
            return SS_ERR_INVALID;
        slots[w.slot].strm = &w;
    }
    for (int k = 0; k < n_streams; ++k)                     // (beyond 2^23 samples a crop's sum need not be exact)
        for (const PoolEntry& e : items[streams[k].slot].pool->host) if (e.N > (1 << 23)) return SS_ERR_UNSUPPORTED;
    return SS_OK;
}

// A plan's background streams (include/sonicsim_b200.h, ss_bg_stream), all but the byte ranges (validate_mixes): the
// record of each bed's slot receives the bed
static int validate_bgs(const ss_ctx* c, const ss_source* items, const ss_bg_stream* bgs, int n_bgs,
                        const ss_plan_draw* draws, int n_draws, std::vector<PlanSlot>& slots) {
    for (int k = 0; k < n_bgs; ++k) {
        const ss_bg_stream& b = bgs[k];
        if (b.slot < 0 || b.slot >= (int)slots.size()) return SS_ERR_INVALID;
        const PlanSlot& r = slots[b.slot];
        if (r.bg || r.strm || r.dry) return SS_ERR_INVALID;
        const ss_pool* pl = items[b.slot].pool;
        // a pooled slot of a pool without loudness gains (a bed has no fixed pair to measure), over a dry pool of this
        // context, with a layout of 1..kStreamEntries aligned device entries
        if (!pl || pl->gains || !b.pool || b.pool->c != c) return SS_ERR_INVALID;
        if (b.m < 1 || b.m > kStreamEntries) return SS_ERR_INVALID;
        for (const int32_t* a : {b.ids_dev, b.offsets_dev, b.heads_dev, b.counts_dev})
            if (!a || ((uintptr_t)a & 3)) return SS_ERR_INVALID;
        for (int j = 0; j < n_draws; ++j)                   // (the draws test speakers only: a bed may be a reader)
            for (int s = 0; s < draws[j].S && s < kDrawSpeakers; ++s)
                if (draws[j].speakers[s] == b.slot) return SS_ERR_INVALID;
        slots[b.slot].bg = &b;
    }
    return SS_OK;
}

// A plan's loudness slots (include/sonicsim_b200.h, ss_stream_lufs), all but the byte ranges (validate_mixes): the
// record of each slot receives its entry.  After validate_streams and validate_bgs, which name the stream and bed slots.
static int validate_lufs(const ss_source* items, const ss_stream_lufs* lufs, int n_lufs, std::vector<PlanSlot>& slots) {
    std::vector<ss_post_lufs> post(n_lufs);
    for (int k = 0; k < n_lufs; ++k) {
        const ss_stream_lufs& q = lufs[k];
        if (q.slot < 0 || q.slot >= (int)slots.size()) return SS_ERR_INVALID;
        const PlanSlot& r = slots[q.slot];
        if (r.lufs || !(r.strm || r.bg) || !q.gating.brk || !q.target_dev || ((uintptr_t)q.target_dev & 7) ||
            ((uintptr_t)q.result_dev & 7))
            return SS_ERR_INVALID;
        for (int j = 0; j < k; ++j) if (lufs[j].slot == q.slot) return SS_ERR_INVALID;
        post[k] = q.gating;
    }
    if (check_post_lufs(post.data(), n_lufs)) return SS_ERR_INVALID;
    for (int k = 0; k < n_lufs; ++k) {
        // a device pool (a whole stem of a host pool would stage every bank row at every run) of one N, C <= 8
        const ss_pool* pl = items[lufs[k].slot].pool;
        if (pl->host_res || pl->C > 8) return SS_ERR_UNSUPPORTED;
        for (const PoolEntry& e : pl->host) if (e.N != pl->host[0].N) return SS_ERR_UNSUPPORTED;
    }
    for (int k = 0; k < n_lufs; ++k) {
        // gating tables inside the whole stem: k_kweight reads samples [brk[0], brk[n_e]), k_loud_gate intervals
        const ss_post_lufs& g = lufs[k].gating;
        const int N = items[lufs[k].slot].pool->host[0].N;
        if (g.brk[0] != 0 || g.brk[g.n_e] > N) return SS_ERR_INVALID;
        for (int e = 0; e < g.n_e; ++e) if (g.brk[e + 1] < g.brk[e]) return SS_ERR_INVALID;
        for (int j = 0; j < g.n_blocks; ++j)
            if (g.blk_lo[j] < 0 || g.blk_hi[j] < g.blk_lo[j] || g.blk_hi[j] > g.n_e) return SS_ERR_INVALID;
    }
    for (int k = 0; k < n_lufs; ++k) slots[lufs[k].slot].lufs = &lufs[k];
    return SS_OK;
}

// A plan's layout draws (include/sonicsim_b200.h, ss_layout_draw) and their speaker groups (ss_layout_group), all but
// the byte ranges (validate_mixes): the record of each drawn slot receives its draw and its groups.  After
// validate_streams and validate_bgs, which name the stream and bed slots.
static int validate_layouts(const ss_layout_draw* layouts, int n_layouts, const ss_layout_group* groups, int n_grouped,
                            std::vector<PlanSlot>& slots) {
    for (int k = 0; k < n_layouts; ++k) {
        const ss_layout_draw& L = layouts[k];
        if (L.slot < 0 || L.slot >= (int)slots.size()) return SS_ERR_INVALID;
        const PlanSlot& r = slots[L.slot];
        if (r.layout || !(r.strm || r.bg) || !L.rng_dev || ((uintptr_t)L.rng_dev & 7) || L.total < 1 ||
            L.sample_rate < 1 || L.sample_rate > INT32_MAX / 10 || (r.strm && L.select_lengths))
            return SS_ERR_INVALID;
        if (L.select_lengths)
            for (int i = 0; i < r.bg->pool->n; ++i) if (L.select_lengths[i] < 0) return SS_ERR_INVALID;
        slots[L.slot].layout = &L;
    }
    // a grouped draw: a stream slot's draw, named once, over bounds that ascend strictly from 0 to its pool's n, with
    // an aligned group_dev
    for (int j = 0; j < n_grouped; ++j) {
        const ss_layout_group& q = groups[j];
        if (q.layout < 0 || q.layout >= n_layouts) return SS_ERR_INVALID;
        const PlanSlot& r = slots[layouts[q.layout].slot];
        if (r.group || !r.strm || q.n_groups < 1 || !q.bounds || !q.group_dev || ((uintptr_t)q.group_dev & 3))
            return SS_ERR_INVALID;
        if (q.bounds[0] != 0 || q.bounds[q.n_groups] != r.strm->pool->n) return SS_ERR_INVALID;
        for (int g = 0; g < q.n_groups; ++g) if (q.bounds[g + 1] <= q.bounds[g]) return SS_ERR_INVALID;
        slots[layouts[q.layout].slot].group = &q;
    }
    for (int k = 0; k < n_layouts; ++k) {
        const PlanSlot& r = slots[layouts[k].slot];
        if (layout_bound(layouts[k], r.clips(), r.bg != nullptr, r.group) > kLayoutCap) return SS_ERR_UNSUPPORTED;
    }
    return SS_OK;
}

// A plan's value draws (include/sonicsim_b200.h, ss_value_draw), all but the byte ranges (validate_value_ranges)
static int validate_values(const ss_value_draw* values, int n_values) {
    if (n_values > kValueDrawsMax) return SS_ERR_UNSUPPORTED;
    std::vector<int64_t> lo(n_values), hi(n_values);    // the least and the most value of each int32 entry
    for (int k = 0; k < n_values; ++k) {
        const ss_value_draw& v = values[k];
        const bool real = v.kind == SS_VALUE_F32 || v.kind == SS_VALUE_F64;
        if (!real && v.kind != SS_VALUE_INT && v.kind != SS_VALUE_DISTINCT) return SS_ERR_INVALID;
        const uintptr_t align = v.kind == SS_VALUE_F64 ? 8 : 4;
        if (!v.out || ((uintptr_t)v.out & (align - 1)) || !v.rng_dev || ((uintptr_t)v.rng_dev & 7))
            return SS_ERR_INVALID;
        if (v.rows < 1 || v.rows > 65535 || v.rows != values[0].rows || v.k < 1 || v.k > 4096) return SS_ERR_INVALID;
        if (real) {
            if (!isfinite(v.low) || !isfinite(v.high) || !(v.low < v.high) || v.base != -1) return SS_ERR_INVALID;
            if (v.kind == SS_VALUE_F32 && ((double)(float)v.low != v.low || (double)(float)v.high != v.high))
                return SS_ERR_INVALID;
            continue;
        }
        const int64_t n = (int64_t)v.ihigh - v.ilow;
        if (n < 1 || (v.kind == SS_VALUE_DISTINCT && (v.k > 64 || v.k > n))) return SS_ERR_INVALID;
        lo[k] = v.ilow;
        hi[k] = (int64_t)v.ihigh - 1;
        if (v.base == -1) continue;
        if (v.base < 0 || v.base >= k || v.stride < 1) return SS_ERR_INVALID;
        const ss_value_draw& b = values[v.base];
        if ((b.kind != SS_VALUE_INT && b.kind != SS_VALUE_DISTINCT) || b.k != 1) return SS_ERR_INVALID;
        lo[k] += lo[v.base] * v.stride;                  // |base| < 2^31 and stride < 2^31: no int64 overflow
        hi[k] += hi[v.base] * v.stride;
        if (lo[k] < INT32_MIN || hi[k] > INT32_MAX) return SS_ERR_INVALID;
    }
    return SS_OK;
}

// The byte ranges of a plan's value draws.  `ranges`: every range the rest of the plan reads or writes
// (validate_mixes).  A value draw's out meets nothing but the small per-run inputs (picks, dry picks, undrawn starts,
// sirs, snr, a draw's u, loudness targets): no other out, no rng, nothing else the plan reads or writes; an rng meets
// nothing the plan writes.
static int validate_value_ranges(const ss_source* items, int n_items, const ss_value_draw* values, int n_values,
                                 std::vector<ByteRange> ranges) {
    if (n_values == 0) return SS_OK;
    ranges.erase(std::remove_if(ranges.begin(), ranges.end(), [](const ByteRange& x) { return x.input; }),
                 ranges.end());
    for (int k = 0; k < n_values; ++k) {
        const ss_value_draw& v = values[k];
        add_range(ranges, v.out, (uint64_t)v.rows * v.k * (v.kind == SS_VALUE_F64 ? 8 : 4), true);
        add_range(ranges, v.rng_dev, 16, false);
        const uintptr_t lo = (uintptr_t)v.rng_dev, hi = lo + 16;  // (the items' outputs count as read ranges)
        for (int i = 0; i < n_items; ++i) {
            const ss_source& it = items[i];
            const uint64_t n_out = 4 * (uint64_t)it.C * (it.win_len > 0 ? it.win_len : it.N);
            for (const float* o : {it.out, (it.flags & SS_DIRECT_TARGET) ? it.out_direct : nullptr})
                if (o && (uintptr_t)o < hi && lo < (uintptr_t)o + n_out) return SS_ERR_INVALID;
        }
    }
    return written_ranges_disjoint(ranges) ? SS_OK : SS_ERR_INVALID;
}

// A plan's trajectories (include/sonicsim_b200.h, ss_trajectory), all but the byte ranges (validate_mixes): the record
// of each trajectory's slot receives it.  After validate_dry_picks, validate_streams and validate_draws: a slot of a
// moving device pool without loudness gains, whose dry pick has no pair gains, and which is no start draw's speaker
// unless it is dry-picked or a stream slot (a speaker's level table is then its dry signal's, not its candidate's stem).
static int validate_trajectories(const ss_source* items, const ss_trajectory* trajs, int n_trajs,
                                 const ss_plan_draw* draws, int n_draws, std::vector<PlanSlot>& slots) {
    for (int k = 0; k < n_trajs; ++k) {
        const ss_trajectory& t = trajs[k];
        if (t.slot < 0 || t.slot >= (int)slots.size() || slots[t.slot].traj) return SS_ERR_INVALID;
        const ss_pool* pl = items[t.slot].pool;
        const PlanSlot& r = slots[t.slot];
        if (!pl || pl->mode != SS_MOVING_BOUNDS || pl->gains || r.pair) return SS_ERR_INVALID;
        if (!t.path_dev || !t.bounds_dev || ((uintptr_t)t.path_dev & 3) || ((uintptr_t)t.bounds_dev & 3))
            return SS_ERR_INVALID;
        if (!r.dry && !r.strm)
            for (int j = 0; j < n_draws; ++j)
                for (int s = 0; s < draws[j].S; ++s) if (draws[j].speakers[s] == t.slot) return SS_ERR_INVALID;
        slots[t.slot].traj = &t;
    }
    for (int k = 0; k < n_trajs; ++k)                       // (a host pool's staging is sized from its host bounds)
        if (items[trajs[k].slot].pool->host_res) return SS_ERR_UNSUPPORTED;
    return SS_OK;
}

// A plan's dereverberation targets (include/sonicsim_b200.h, ss_plan_target), all but the speakers' direct-path stems
// and the byte ranges (validate_mixes): mix receives the mixtures, each with its target's direct_out, or null
static int validate_targets(const ss_plan_mix* mixes, int n_mixes, const ss_plan_target* targets, int n_targets,
                            std::vector<PlanMix>& mix) {
    for (int k = 0; k < n_mixes; ++k) mix.push_back({mixes[k], nullptr});
    for (int j = 0; j < n_targets; ++j) {
        const ss_plan_target& t = targets[j];
        if (t.mix < 0 || t.mix >= n_mixes || mix[t.mix].dir_out || !t.direct_out) return SS_ERR_INVALID;
        mix[t.mix].dir_out = t.direct_out;
    }
    return SS_OK;
}

// Every ss_plan_create* export.  A call refused for its arguments leaves *out untouched; a later failure leaves it null.
static int plan_create(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                       const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                       const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                       int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                       const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts, int n_layouts,
                       const ss_value_draw* values, int n_values, const ss_layout_group* groups, int n_grouped,
                       const ss_trajectory* trajs, int n_trajs, ss_plan** out) {
    auto bad = [](const void* a, int n) { return n < 0 || (n > 0 && !a); };   // an array and its count
    if (!c || !out || !items || n_items <= 0 || bad(mixes, n_mixes) || bad(draws, n_draws) || bad(picks, n_picks) ||
        bad(targets, n_targets) || bad(streams, n_streams) || bad(bgs, n_bgs) || bad(lufs, n_lufs) ||
        bad(layouts, n_layouts) || bad(values, n_values) || bad(groups, n_grouped) || bad(trajs, n_trajs))
        return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    std::vector<Shape> shapes;
    std::vector<PlanSlot> slots(n_items);
    std::vector<PlanMix> mix;
    { int st = shape_dev_items(c, items, n_items, shapes, true); if (st) return st; }
    { int st = validate_dry_picks(c, items, picks, pair_gains, n_picks, slots); if (st) return st; }
    { int st = validate_streams(c, items, streams, n_streams, slots); if (st) return st; }
    { int st = validate_bgs(c, items, bgs, n_bgs, draws, n_draws, slots); if (st) return st; }
    { int st = validate_lufs(items, lufs, n_lufs, slots); if (st) return st; }
    { int st = validate_layouts(layouts, n_layouts, groups, n_grouped, slots); if (st) return st; }
    { int st = validate_values(values, n_values); if (st) return st; }
    { int st = validate_draws(items, slots, draws, n_draws); if (st) return st; }
    { int st = validate_trajectories(items, trajs, n_trajs, draws, n_draws, slots); if (st) return st; }
    { int st = validate_targets(mixes, n_mixes, targets, n_targets, mix); if (st) return st; }
    std::vector<ByteRange> ranges;
    { int st = validate_mixes(items, slots, mix, draws, n_draws, ranges); if (st) return st; }
    { int st = validate_value_ranges(items, n_items, values, n_values, std::move(ranges)); if (st) return st; }
    *out = nullptr;
    ss_plan* p = new (std::nothrow) ss_plan();
    if (!p) return SS_ERR_NOMEM;
    p->c = c;
    for (int i = 0; i < n_items; ++i) {
        ss_bank* b = const_cast<ss_bank*>(items[i].rir_bank);
        if (b && std::find(p->banks.begin(), p->banks.end(), b) == p->banks.end()) p->banks.push_back(b);
        ss_pool* pl = const_cast<ss_pool*>(items[i].pool);
        if (pl && std::find(p->pools.begin(), p->pools.end(), pl) == p->pools.end()) p->pools.push_back(pl);
    }
    const int st = plan_build(p, items, shapes.data(), slots, mix, draws, n_draws, layouts, n_layouts, values,
                              n_values, groups, n_grouped);
    if (st != SS_OK) { ss_plan_destroy(p); return st; }
    for (ss_pool* pl : p->pools) pl->planned = true;   // its descriptors hold the pool's gain pointer (ss_pool_loudness)
    *out = p;
    return SS_OK;
}

extern "C" int ss_plan_create(ss_ctx* c, const ss_source* items, int n_items, ss_plan** out) {
    return plan_create(c, items, n_items, nullptr, 0, nullptr, 0, nullptr, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0,
                       nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_mix(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                  int n_mixes, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, nullptr, 0, nullptr, nullptr, 0, nullptr, 0, nullptr, 0, nullptr,
                       0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_ex(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                 int n_mixes, const ss_plan_draw* draws, int n_draws, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, nullptr, nullptr, 0, nullptr, 0, nullptr, 0,
                       nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_pair(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                   int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                   const ss_pair_gains* const* pair_gains, int n_picks, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, nullptr, 0, nullptr,
                       0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_target(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                     int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                     const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                     int n_targets, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_stream(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                     int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                     const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                     int n_targets, const ss_dry_stream* streams, int n_streams, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_bg(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                                 const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                 const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                 int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs,
                                 int n_bgs, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, bgs, n_bgs, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_lufs(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                   int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                   const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                   int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs,
                                   int n_bgs, const ss_stream_lufs* lufs, int n_lufs, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, bgs, n_bgs, lufs, n_lufs, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_layout(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                     int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                     const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                     int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs,
                                     int n_bgs, const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts,
                                     int n_layouts, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, bgs, n_bgs, lufs, n_lufs, layouts, n_layouts, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_values(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                     int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                     const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                     int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs,
                                     int n_bgs, const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts,
                                     int n_layouts, const ss_value_draw* values, int n_values, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, bgs, n_bgs, lufs, n_lufs, layouts, n_layouts, values, n_values, nullptr, 0,
                       nullptr, 0, out);
}

extern "C" int ss_plan_create_groups(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                     int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                     const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                     int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs,
                                     int n_bgs, const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts,
                                     int n_layouts, const ss_value_draw* values, int n_values,
                                     const ss_layout_group* groups, int n_grouped, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, bgs, n_bgs, lufs, n_lufs, layouts, n_layouts, values, n_values, groups,
                       n_grouped, nullptr, 0, out);
}

extern "C" int ss_plan_create_dry(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                  int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                  int n_picks, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, nullptr, n_picks, nullptr, 0, nullptr, 0,
                       nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, nullptr, 0, out);
}

extern "C" int ss_plan_create_traj(ss_ctx* c, const ss_source* items, int n_items, const ss_plan_mix* mixes,
                                   int n_mixes, const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                                   const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                                   int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs,
                                   int n_bgs, const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts,
                                   int n_layouts, const ss_value_draw* values, int n_values,
                                   const ss_layout_group* groups, int n_grouped, const ss_trajectory* trajs,
                                   int n_trajs, ss_plan** out) {
    return plan_create(c, items, n_items, mixes, n_mixes, draws, n_draws, picks, pair_gains, n_picks, targets, n_targets,
                       streams, n_streams, bgs, n_bgs, lufs, n_lufs, layouts, n_layouts, values, n_values, groups,
                       n_grouped, trajs, n_trajs, out);
}

// The start draws (k_draw) on `stream`, ahead of everything that reads a start
static int draw_enqueue(ss_ctx* c, const DrawDesc* d, int n, bool i16, bool streams, cudaStream_t stream) {
    if (streams) k_draw<true, true><<<(n + 3) / 4, 128, 0, stream>>>(d, n);
    else if (i16) k_draw<true><<<(n + 3) / 4, 128, 0, stream>>>(d, n);
    else k_draw<false><<<(n + 3) / 4, 128, 0, stream>>>(d, n);
    CK(cudaGetLastError());
    c->launches += 1;
    return SS_OK;
}

// the value draws (whose values everything after them may read), the layout draws, the start draws (which walk stream
// layouts), the host-pool staging, the launches of every chunk
// (run_chunks), the loudness slots' measurements and crops, then the mixtures (which read every chunk's outputs and the
// crops) on `stream`
static int plan_enqueue(ss_plan* p, cudaStream_t stream) {
    ss_ctx* c = p->c;
    if (p->n_value) {
        k_values<<<(p->value_rows + kValueWarps - 1) / kValueWarps, 32 * kValueWarps, 0, stream>>>(p->d_value, p->n_value,
                                                                                                p->value_rows);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    if (p->n_layout) {
        if (p->d_layout_group)
            k_layout_grouped<<<p->n_layout, 32, p->layout_smem, stream>>>(p->d_layout, p->d_layout_group);
        else
            k_layout<<<p->n_layout, 32, p->layout_smem, stream>>>(p->d_layout);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    if (p->n_draw) {
        const int st = draw_enqueue(c, p->d_draw, p->n_draw, p->draw16, p->draw_stream, stream);
        if (st) return st;
    }
    if (p->n_stage) {                                   // staged slots: after the draws, before any chunk reads a slot
        const dim3 grid(kStageCtas, p->n_stage);
        if (p->n_tap && p->stage_bg) k_stage<true, true, true, true><<<grid, 256, 0, stream>>>(p->d_stage, p->d_taps);
        else if (p->stage_bg) k_stage<true, false, true, true><<<grid, 256, 0, stream>>>(p->d_stage, nullptr);
        else if (p->n_tap && p->stage_stream) k_stage<true, true, true><<<grid, 256, 0, stream>>>(p->d_stage, p->d_taps);
        else if (p->stage_stream) k_stage<true, false, true><<<grid, 256, 0, stream>>>(p->d_stage, nullptr);
        else if (p->n_tap && p->stage16) k_stage<true, true><<<grid, 256, 0, stream>>>(p->d_stage, p->d_taps);
        else if (p->n_tap) k_stage<false, true><<<grid, 256, 0, stream>>>(p->d_stage, p->d_taps);
        else if (p->stage16) k_stage<true><<<grid, 256, 0, stream>>>(p->d_stage, nullptr);
        else k_stage<false><<<grid, 256, 0, stream>>>(p->d_stage, nullptr);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    if (p->n_tap) {                                     // the staged tap rows into the spectra the slots' views name
        static const PrepParams global_tables = {};     // (n_inline = 0: the Sources k_stage wrote, from global memory)
        k_prepare<false><<<p->tap_ctas, kThreads, kPadF * (int)sizeof(float2), stream>>>(
            p->d_tap_src, p->d_tap_prefix, p->n_tap, nullptr, global_tables);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    const int rc = run_chunks(c, p->chunks.size(), stream, p->ev_fork, p->ev_join, [&](size_t k, cudaStream_t s, int) {
        return chunk_enqueue(c, p->chunks[k], s, c->profiling);
    });
    if (rc) return rc;
    if (p->n_loud) {                                    // loudness slots: measure the whole stems, then cut the crops
        const int st = loud_measure_enqueue(c, p->d_loud, p->d_loud_prefix, p->n_loud, p->loud_total, p->loud_rate, stream);
        if (st) return st;
        k_loud_crop<<<dim3(p->crop_ctas, p->n_loud), 256, 0, stream>>>(p->d_crop);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    return p->n_mix ? mix_enqueue(c, p->d_mix, p->n_mix, stream, p->mix_direct) : SS_OK;
}

extern "C" int ss_plan_run(ss_plan* p, void* stream_) {
    if (!p) return SS_ERR_INVALID;
    ss_ctx* c = p->c;
    cudaStream_t stream = (cudaStream_t)stream_;
    CK(cudaSetDevice(c->device));
    for (ss_bank* b : p->banks) CK(cudaStreamWaitEvent(stream, b->ready, 0));    // (outside any capture)
    for (ss_pool* pl : p->pools) CK(cudaStreamWaitEvent(stream, pl->ready, 0));
    if (c->profiling) {                                 // per-kernel timing: no graph, chunks one after the other
        { int st = profile_start(c, stream); if (st) return st; }
        return plan_enqueue(p, stream);
    }
    if (!p->exec && !p->graph_failed && !c->no_graph) {
        const int64_t launches_before = c->launches;
        cudaGraph_t g = nullptr;
        bool ok = cudaStreamBeginCapture(p->s_cap, cudaStreamCaptureModeThreadLocal) == cudaSuccess;
        if (ok) {
            const int st = plan_enqueue(p, p->s_cap);
            const cudaError_t e = cudaStreamEndCapture(p->s_cap, &g);
            ok = st == SS_OK && e == cudaSuccess && g != nullptr;
        }
        if (ok) ok = cudaGraphInstantiate(&p->exec, g, 0) == cudaSuccess;
        if (g) cudaGraphDestroy(g);
        p->launches_per_run = (int)(c->launches - launches_before);      // what the graph launches at every run ...
        c->launches = launches_before;                                    // ... none of which ran while capturing
        if (!ok) { p->exec = nullptr; p->graph_failed = true; (void)cudaGetLastError(); }
    }
    if (p->exec) {
        CK(cudaGraphLaunch(p->exec, stream));
        c->launches += p->launches_per_run;
        return SS_OK;
    }
    return plan_enqueue(p, stream);
}
// 1: the plan runs as an instantiated CUDA graph, 0: not (yet), negative: error
extern "C" int ss_plan_is_graph(const ss_plan* p) { return p ? (p->exec ? 1 : 0) : SS_ERR_INVALID; }

// ----------------------------------------------------------------------------- host path
// What the host path copies in and out for one source: dry samples [xa, xb), RIR positions [pa, pb], idx / w entries
// [ia, ib), and C * wl output floats per stem - the whole source, or a windowed source's read set (window_shape)
struct ReadSet { int xa, xb, pa, pb, ia, ib, wl; };
static ReadSet read_set(const ss_source& it, const Shape& sh) {
    ReadSet r = {0, it.N, 0, it.P - 1, 0, it.N, it.N};
    if (sh.win) { r.xa = sh.xa; r.xb = sh.xb; r.pa = sh.pa; r.pb = sh.pb; r.ia = sh.ia; r.ib = sh.ib; r.wl = it.win_len; }
    return r;
}
// idx (SS_MOVING_INDEXED): the entries the render reads (the bounds table is checked whole, before read_set plans from it)
static int check_idx_host(const ss_source& it, const ReadSet& rs) {
    if (it.mode == SS_MOVING_INDEXED)
        for (int n = rs.ia; n < rs.ib; ++n) { int v = it.idx[n]; if (v < 0 || v + 1 >= it.P) return SS_ERR_INDEX; }
    return SS_OK;
}

// Where one source's arrays go in its chunk's slot: its inputs (x, rir, bounds or idx, w) in d_in and its outputs
// (out, out_direct, loudness scratch and result) in d_out, each at a 256-byte boundary after the chunk's earlier
// arrays, which end at *in / *out.  An array the source does not stage has 0 bytes.
struct Span { size_t at, bytes; };
struct Staged { Span x, rir, tab, w, out, direct, scratch, res; };
static Staged stage_source(const ss_source& it, const ReadSet& rs, const ss_post_lufs* q, size_t* in, size_t* out) {
    auto take = [](size_t* end, size_t bytes) { const Span s = {*end, bytes}; *end += align_up(bytes, 256); return s; };
    Staged s = {};
    s.x = take(in, sizeof(float) * (size_t)(rs.xb - rs.xa));
    if (!it.rir_bank) s.rir = take(in, sizeof(float) * (size_t)(rs.pb - rs.pa + 1) * it.C * it.L);
    if (it.mode == SS_MOVING_BOUNDS) s.tab = take(in, sizeof(int32_t) * (size_t)it.P);
    if (it.mode == SS_MOVING_INDEXED) { s.tab = take(in, 4 * (size_t)(rs.ib - rs.ia)); s.w = take(in, s.tab.bytes); }
    s.out = take(out, sizeof(float) * (size_t)it.C * rs.wl);
    if (it.flags & SS_DIRECT_TARGET) s.direct = take(out, s.out.bytes);
    if (q) { s.scratch = take(out, loud_scratch_bytes(*q, it.C)); s.res = take(out, 2 * sizeof(double)); }
    return s;
}

// Host path: H2D -> k_spectra -> k_render [-> loudness measure + in-place gain] -> D2H, pipelined
// over chunks on three streams with two device slots.
extern "C" int ss_render_host_ex(ss_ctx* c, const ss_source* items, int n_items, const ss_post_lufs* post) {
    if (!c || (!items && n_items > 0) || n_items < 0) return SS_ERR_INVALID;
    if (n_items == 0) return SS_OK;
    CK(cudaSetDevice(c->device));
    if (post && check_post_lufs(post, n_items)) return SS_ERR_INVALID;
    std::vector<Shape> shapes(n_items);
    std::vector<ReadSet> rset(n_items);
    for (int i = 0; i < n_items; ++i) {
        int st = validate_item_ctx(c, items[i]); if (st) return st;
        // a window cannot be loudness-normalised: the reference measures the whole stem
        if (post && post[i].brk && items[i].win_len > 0) return SS_ERR_INVALID;
        // a moving window's read set depends on a start that only the device knows
        if (items[i].win_start_dev) return SS_ERR_INVALID;
        if (items[i].mode == SS_MOVING_BOUNDS && !bounds_ok(items[i].bounds, items[i].P, items[i].N)) return SS_ERR_INVALID;
        // planned as it is rendered: with the trajectory in host memory (bounds_host = bounds, as below)
        ss_source h = items[i];
        if (h.mode == SS_MOVING_BOUNDS) h.bounds_host = h.bounds;
        shapes[i] = shape_of(h);
        rset[i] = read_set(items[i], shapes[i]);
        st = check_idx_host(items[i], rset[i]); if (st) return st;
        if (post && post[i].brk && items[i].C > 8) return SS_ERR_INVALID;
    }
    // an earlier asynchronous ss_render_dev may still be using scratch buffer 0 on its internal streams
    for (int i = 0; i < ss_ctx::kAux; ++i) CK(cudaStreamWaitEvent(c->s_cmp, c->ev_join[i], 0));
    // banks built asynchronously on the caller's stream: every render of this call (on s_cmp) comes after them
    { int st = wait_banks(items, n_items, c->s_cmp); if (st) return st; }
    std::vector<int> cuts;
    make_chunks(items, shapes.data(), n_items, c->chunk_bytes_host, cuts);
    std::vector<ss_source> dev(n_items);
    std::vector<Staged> staged(n_items);
    std::vector<ss_loud_item> loud;
    std::vector<ScaleItem> direct_gain;                  // direct-path stems scaled by their reverberant stem's gain
    std::vector<double*> res_dev(n_items, nullptr);
    // loudness: (a) the gating tables of all sources that share them (same host arrays = same clip length, the normal
    // case) are uploaded once per call from a pinned staging copy; (b) the two result doubles of every stem come back
    // into pinned memory - a copy into the caller's pageable array would block the host until the stream gets
    // there and serialise the whole pipeline; (c) the loudness kernels of consecutive chunks run on rotating side
    // streams: their grids are small and latency-bound, three of them overlap each other, the
    // next chunk's render and the copies
    GatingTables tabs;
    const size_t res_bytes = align_up(2 * sizeof(double) * (size_t)n_items, 256);   // [0, res_bytes): results
    if (post) {
        tabs = gating_tables(post, n_items);
        const size_t tab_bytes = tabs.bytes.size();
        { const int st = ensure_pair(&c->h_post, &c->d_post, &c->h_post_cap, tab_bytes + res_bytes); if (st) return st; }
        char* const h_tab = c->h_post + res_bytes;
        if (tab_bytes) {
            memcpy(h_tab, tabs.bytes.data(), tab_bytes);
            CK(cudaMemcpyAsync(c->d_post + res_bytes, h_tab, tab_bytes, cudaMemcpyHostToDevice, c->s_in));
        }
    }
    double* const h_res = post ? (double*)c->h_post : nullptr;
    const char* const d_tab = post ? c->d_post + res_bytes : nullptr;
    // the pipeline proper; any failure falls through to the stream synchronisation below, so that no copy is
    // still reading or writing the caller's buffers when this function returns
    auto pipeline = [&]() -> int {
    int rc = SS_OK;
    for (size_t k = 0; k + 1 < cuts.size() && rc == SS_OK; ++k) {
        const int first = cuts[k], last = cuts[k + 1];
        ss_ctx::Slot& sl = c->slot[k % ss_ctx::kSlots];
        size_t in_b = 0, out_b = 0;
        for (int i = first; i < last; ++i)
            staged[i] = stage_source(items[i], rset[i], post && post[i].brk ? &post[i] : nullptr, &in_b, &out_b);
        if (k >= (size_t)ss_ctx::kSlots) CK(cudaEventSynchronize(sl.ev_free));      // slot's previous chunk fully drained
        if ((rc = ensure(&sl.d_in, &sl.in_cap, in_b)) != SS_OK) break;
        if ((rc = ensure(&sl.d_out, &sl.out_cap, out_b)) != SS_OK) break;
        char* const pi = sl.d_in; char* const po = sl.d_out;
        loud.clear();
        direct_gain.clear();
        for (int i = first; i < last; ++i) {
            const ss_source& it = items[i];
            const ReadSet& rs = rset[i];
            const Staged& s = staged[i];
            ss_source d = it;
            // only the read set is copied; the device pointers are offset so that the kernels index the full arrays
            CK(cudaMemcpyAsync(pi + s.x.at, it.x + rs.xa, s.x.bytes, cudaMemcpyHostToDevice, c->s_in));
            d.x = (const float*)(pi + s.x.at) - rs.xa;
            if (!it.rir_bank) {                              // a banked source's spectra are on the device already
                const size_t pos0 = (size_t)rs.pa * it.C * it.L;
                CK(cudaMemcpyAsync(pi + s.rir.at, it.rir + pos0, s.rir.bytes, cudaMemcpyHostToDevice, c->s_in));
                d.rir = (const float*)(pi + s.rir.at) - pos0;
            }
            if (it.mode == SS_MOVING_BOUNDS) {
                CK(cudaMemcpyAsync(pi + s.tab.at, it.bounds, s.tab.bytes, cudaMemcpyHostToDevice, c->s_in));
                d.bounds = (const int32_t*)(pi + s.tab.at);
                d.bounds_host = it.bounds;
            } else if (it.mode == SS_MOVING_INDEXED) {
                CK(cudaMemcpyAsync(pi + s.tab.at, it.idx + rs.ia, s.tab.bytes, cudaMemcpyHostToDevice, c->s_in));
                CK(cudaMemcpyAsync(pi + s.w.at, it.w + rs.ia, s.w.bytes, cudaMemcpyHostToDevice, c->s_in));
                d.idx = (const int32_t*)(pi + s.tab.at) - rs.ia; d.w = (const float*)(pi + s.w.at) - rs.ia;
            }
            d.out = (float*)(po + s.out.at);
            if (it.flags & SS_DIRECT_TARGET) d.out_direct = (float*)(po + s.direct.at);
            dev[i] = d;
            if (post && post[i].brk) {
                double* const scratch = (double*)(po + s.scratch.at);
                res_dev[i] = (double*)(po + s.res.at);
                loud.push_back(loud_item(post[i], d_tab + tabs.at[i], d.out, d.out, it.N, it.C, scratch, res_dev[i]));
                if (it.flags & SS_DIRECT_TARGET) direct_gain.push_back(ScaleItem{d.out_direct, res_dev[i], it.N, it.C});
            }
        }
        CK(cudaEventRecord(sl.ev_in, c->s_in));
        CK(cudaStreamWaitEvent(c->s_cmp, sl.ev_in, 0));
        rc = launch_chunk(c, dev.data(), shapes.data(), first, last, c->s_cmp, 0);
        if (rc != SS_OK) break;
        if (!loud.empty()) {
            cudaStream_t s_l = c->s_aux[k % ss_ctx::kAux];
            CK(cudaEventRecord(sl.ev_rend, c->s_cmp));
            CK(cudaStreamWaitEvent(s_l, sl.ev_rend, 0));
            rc = ss_loudness_dev(c, loud.data(), (int)loud.size(), (void*)s_l);
            if (rc != SS_OK) break;
            rc = loud_scale_dev(c, direct_gain.data(), (int)direct_gain.size(), s_l);
            if (rc != SS_OK) break;
            CK(cudaEventRecord(sl.ev_done, s_l));
        } else {
            CK(cudaEventRecord(sl.ev_done, c->s_cmp));
        }
        CK(cudaStreamWaitEvent(c->s_out, sl.ev_done, 0));
        for (int i = first; i < last; ++i) {
            const Staged& s = staged[i];
            CK(cudaMemcpyAsync(items[i].out, dev[i].out, s.out.bytes, cudaMemcpyDeviceToHost, c->s_out));
            if (items[i].flags & SS_DIRECT_TARGET)
                CK(cudaMemcpyAsync(items[i].out_direct, dev[i].out_direct, s.direct.bytes, cudaMemcpyDeviceToHost, c->s_out));
            if (res_dev[i])
                CK(cudaMemcpyAsync(h_res + 2 * i, res_dev[i], s.res.bytes, cudaMemcpyDeviceToHost, c->s_out));
        }
        CK(cudaEventRecord(sl.ev_free, c->s_out));
        // the next chunk's H2D into the *other* slot may start now; it must not overtake the
        // render still reading this slot, which the per-slot ev_free wait above guarantees.
    }
    return rc;
    };
    const int rc = pipeline();
    cudaError_t e1 = cudaStreamSynchronize(c->s_in), e2 = cudaStreamSynchronize(c->s_cmp), e3 = cudaSuccess;
    if (post) for (int i = 0; i < ss_ctx::kAux; ++i) { cudaError_t e = cudaStreamSynchronize(c->s_aux[i]); if (e3 == cudaSuccess) e3 = e; }
    cudaError_t e4 = cudaStreamSynchronize(c->s_out);
    if (rc != SS_OK) return rc;
    CK(e1); CK(e2); CK(e3); CK(e4);
    if (post)
        for (int i = 0; i < n_items; ++i)
            if (res_dev[i] && post[i].result) { post[i].result[0] = h_res[2 * i]; post[i].result[1] = h_res[2 * i + 1]; }
    return SS_OK;
}

extern "C" int ss_render_host(ss_ctx* c, const ss_source* items, int n_items) {
    return ss_render_host_ex(c, items, n_items, nullptr);
}

extern "C" int ss_convolve_fixed_receiver(ss_ctx* c, const float* x, const float* rirs, float* out,
                                          int32_t N, int32_t C, int32_t L) {
    ss_source it; memset(&it, 0, sizeof(it));
    it.x = x; it.rir = rirs; it.out = out; it.N = N; it.P = 1; it.C = C; it.L = L; it.mode = SS_STATIC;
    return ss_render_host(c, &it, 1);
}
extern "C" int ss_convolve_moving_receiver(ss_ctx* c, const float* x, const float* rirs, const int32_t* idx,
                                           const float* w, float* out, int32_t N, int32_t P, int32_t C, int32_t L) {
    ss_source it; memset(&it, 0, sizeof(it));
    it.x = x; it.rir = rirs; it.out = out; it.idx = idx; it.w = w;
    it.N = N; it.P = P; it.C = C; it.L = L; it.mode = SS_MOVING_INDEXED;
    return ss_render_host(c, &it, 1);
}
