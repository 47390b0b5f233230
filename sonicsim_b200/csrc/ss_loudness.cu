// sonicsim_b200 :: ss_loudness.cu - SonicSim_audio.lufs_norm (SonicSim_audio.py:68-81) on the GPU.
//   k_kweight<1,2,3> : one thread per (stem, channel, elementary interval); three passes over the thread's own interval,
//   k_kw_scan          with a warp-parallel scan of the per-interval state maps between them, give the exact filter state at
//                      every interval's start (ss_loud.cuh) and the energy of the K-weighted signal
//   k_loud_gate      : one CTA per stem: block loudness, absolute / relative gates (fixed-order reductions), LUFS, gain
//   k_loud_scale     : out = gain * data (float4 vectorised)
#include <math.h>
#include <string.h>

#include <algorithm>

#include "ss_internal.h"
#include "ss_loud.cuh"

using namespace ss;

static_assert(kLoudScratch == SS_LOUD_SCRATCH_DOUBLES, "scratch contract of include/sonicsim_b200.h");

// One thread per (stem, channel, elementary interval), a warp = 32 consecutive work items.  Every thread walks its
// own interval sequentially (the recurrence), so reading the samples directly would touch 32 different cache lines per
// load instruction; instead the warp moves 32 x 32-sample tiles through shared memory: row r of the tile is loaded by
// all lanes at once (128 contiguous bytes of work item r's interval when the stem is channel-major), then lane j
// consumes row j.
template <int PASS>
__global__ void __launch_bounds__(128)
k_kweight(const LoudItem* __restrict__ items, const int* __restrict__ prefix, int n_items, KCoef k) {
    __shared__ float tile[4][32][33];
    __shared__ const float* row_ptr[4][32];           // first sample of work item r's interval
    __shared__ int row_len[4][32];
    __shared__ long long row_stride[4][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int gid = blockIdx.x * blockDim.x + threadIdx.x;
    const bool live = gid < prefix[n_items];
    int lo = 0, c = 0, e = 0, len = 0;
    row_ptr[warp][lane] = nullptr; row_len[warp][lane] = 0; row_stride[warp][lane] = 1;
    if (live) {
        int hi = n_items - 1;
        while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (prefix[mid] <= gid) lo = mid; else hi = mid - 1; }
        const LoudItem& it = items[lo];
        const int local = gid - prefix[lo];
        c = local / it.n_e; e = local - c * it.n_e;
        const int start = it.brk[e];
        len = it.brk[e + 1] - start;
        row_ptr[warp][lane] = it.data + (long long)c * it.stride_c + (long long)start * it.stride_n;
        row_len[warp][lane] = len;
        row_stride[warp][lane] = it.stride_n;
    }
    KwState st;
    if (live) kw_begin<PASS>(items[lo], c, e, st);
    // longest interval of the warp decides the trip count (intervals are 0.1 s, the last of a stem may be shorter)
    int maxlen = len;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const int v = __shfl_xor_sync(0xffffffffu, maxlen, o); maxlen = v > maxlen ? v : maxlen; }
    __syncwarp();
    // lane l fetches sample s0 + l of every row r: 128 contiguous bytes per row for a channel-major stem
    float nxt[32];
    auto fetch = [&](int s0) {
#pragma unroll
        for (int r = 0; r < 32; ++r) {
            const int n = s0 + lane;
            nxt[r] = n < row_len[warp][r] ? row_ptr[warp][r][(long long)n * row_stride[warp][r]] : 0.f;
        }
    };
    fetch(0);
    for (int s0 = 0; s0 < maxlen; s0 += 32) {
#pragma unroll
        for (int r = 0; r < 32; ++r) tile[warp][r][lane] = nxt[r];
        __syncwarp();
        if (s0 + 32 < maxlen) fetch(s0 + 32);          // in flight while this tile is consumed
        const int cnt = len - s0 < 32 ? len - s0 : 32;
        if (live) for (int i = 0; i < cnt; ++i) kw_sample<PASS>(k, tile[warp][lane][i], st);
        __syncwarp();
    }
    if (live) kw_end<PASS>(items[lo], k, c, e, st);
}

// States at the start of every interval of one (stem, channel): S_(e+1) = M_e S_e + F_e is a scan over affine maps
// x -> A x + b.  One warp per (stem, channel): every lane composes the maps of its own run of intervals, the 32
// composites are scanned with shuffles (composition is associative), then every lane walks its run again from the
// state it starts in and stores the per-interval states.
__global__ void __launch_bounds__(32) k_kw_scan(const LoudItem* __restrict__ items, int stage) {
    const LoudItem& it = items[blockIdx.y];
    const int c = blockIdx.x, lane = threadIdx.x;
    if (c >= it.C) return;
    const int wm = stage ? 5 : 4, wf = stage ? 3 : 1, ws = stage ? 6 : 2;
    const int chunk = (it.n_e + 31) / 32;
    const int e0 = lane * chunk < it.n_e ? lane * chunk : it.n_e, e1 = e0 + chunk < it.n_e ? e0 + chunk : it.n_e;
    // composite of the lane's own run: x -> A x + b
    double a00 = 1, a01 = 0, a10 = 0, a11 = 1, b0 = 0, b1 = 0;
    for (int e = e0; e < e1; ++e) {
        const double* m = loud_slot(it, wm, c, e);
        const double* f = loud_slot(it, wf, c, e);
        const double n00 = m[0] * a00 + m[1] * a10, n01 = m[0] * a01 + m[1] * a11;
        const double n10 = m[2] * a00 + m[3] * a10, n11 = m[2] * a01 + m[3] * a11;
        const double nb0 = m[0] * b0 + m[1] * b1 + f[0], nb1 = m[2] * b0 + m[3] * b1 + f[1];
        a00 = n00; a01 = n01; a10 = n10; a11 = n11; b0 = nb0; b1 = nb1;
    }
    // inclusive scan over the lanes: (A, b) := (A, b) o (A', b') of the lane `o` below = (A A', A b' + b)
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double p00 = __shfl_up_sync(0xffffffffu, a00, o), p01 = __shfl_up_sync(0xffffffffu, a01, o);
        const double p10 = __shfl_up_sync(0xffffffffu, a10, o), p11 = __shfl_up_sync(0xffffffffu, a11, o);
        const double q0 = __shfl_up_sync(0xffffffffu, b0, o), q1 = __shfl_up_sync(0xffffffffu, b1, o);
        if (lane >= o) {
            const double n00 = a00 * p00 + a01 * p10, n01 = a00 * p01 + a01 * p11;
            const double n10 = a10 * p00 + a11 * p10, n11 = a10 * p01 + a11 * p11;
            const double nb0 = a00 * q0 + a01 * q1 + b0, nb1 = a10 * q0 + a11 * q1 + b1;
            a00 = n00; a01 = n01; a10 = n10; a11 = n11; b0 = nb0; b1 = nb1;
        }
    }
    // state the lane's run starts in = what the maps of all lower lanes make of the rest state
    double z1 = __shfl_up_sync(0xffffffffu, b0, 1), z2 = __shfl_up_sync(0xffffffffu, b1, 1);
    if (lane == 0) { z1 = 0; z2 = 0; }
    for (int e = e0; e < e1; ++e) {
        double* s = loud_slot(it, ws, c, e);
        s[0] = z1; s[1] = z2;
        const double* m = loud_slot(it, wm, c, e);
        const double* f = loud_slot(it, wf, c, e);
        const double n1 = m[0] * z1 + m[1] * z2 + f[0], n2 = m[2] * z1 + m[3] * z2 + f[1];
        z1 = n1; z2 = n2;
    }
}

// Gating (pyloudnorm meter.py integrated_loudness; ss_loud.cuh loudness_gate is the one-thread statement of it that the
// CPU emulation runs): one CTA per stem, the gating blocks dealt to its threads, per-channel sums over the blocks that
// pass a gate reduced in a fixed order (warp shuffles, then the warps in turn) so that runs are bit-reproducible.
constexpr int kGateThreads = 128;
__device__ __forceinline__ double gate_reduce(double v, double* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double r = 0;
    for (int w = 0; w < kGateThreads / 32; ++w) r += sh[w];
    return r;                                            // the same value in every thread
}
// k_loud_gate<true> (the loudness slots of plans) reads each item's target from target_dev at every run
// (loud_result_dev): a non-finite target gives the gain NaN.
template <bool DEV_TARGET = false>
__global__ void __launch_bounds__(kGateThreads) k_loud_gate(const LoudItem* __restrict__ items, int n_items) {
    __shared__ double sh[kGateThreads / 32];
    const LoudItem& it = items[blockIdx.x];
    const int nb = it.n_blocks, C = it.C;
    double zmean[8];
    double gamma_r = 0;
    for (int pass = 0; pass < 2; ++pass) {
        double zs[8], cnt = 0;
#pragma unroll
        for (int c = 0; c < 8; ++c) zs[c] = 0;
        for (int j = threadIdx.x; j < nb; j += kGateThreads) {
            double zc[8], s = 0;
#pragma unroll
            for (int c = 0; c < 8; ++c) {
                if (c < C) {
                    double z = 0;
                    for (int e = it.blk_lo[j]; e < it.blk_hi[j]; ++e) z += it.E[(long long)c * it.n_e + e];
                    zc[c] = z * it.inv_norm;
                    s += channel_gain(c) * zc[c];
                }
            }
            const double l = -0.691 + 10.0 * log10(s);
            const bool ok = pass == 0 ? (l >= -70.0) : (l > gamma_r && l > -70.0);
            if (ok) {
#pragma unroll
                for (int c = 0; c < 8; ++c) if (c < C) zs[c] += zc[c];
                cnt += 1.0;
            }
        }
        const double n_ok = gate_reduce(cnt, sh);
        double s = 0;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
            if (c < C) {
                const double tot = gate_reduce(zs[c], sh);
                // pass 0: mean of an empty list is NaN (nothing passes the relative gate then); pass 1: nan_to_num -> 0
                zmean[c] = n_ok > 0 ? tot / n_ok : (pass == 0 ? NAN : 0.0);
                s += channel_gain(c) * zmean[c];
            }
        }
        if (pass == 0) gamma_r = -0.691 + 10.0 * log10(s) - 10.0;
        else if (threadIdx.x == 0) {
            const double lufs = -0.691 + 10.0 * log10(s);                      // log10(0) = -inf
            if (DEV_TARGET) { loud_result_dev(lufs, *it.target_dev, it.result); return; }
            const double used = isinf(lufs) ? -40.0 : lufs;                     // SonicSim_audio.py:73-75
            it.result[0] = lufs;
            it.result[1] = pow(10.0, (it.target - used) / 20.0);               // pyln.normalize.loudness
        }
    }
}

__global__ void __launch_bounds__(256)
k_loud_scale(const LoudItem* __restrict__ items) {
    const LoudItem& it = items[blockIdx.y];
    if (!it.out) return;
    const float g = (float)it.result[1];
    const long long total = (long long)it.N * it.C;
    const long long stride = (long long)gridDim.x * blockDim.x;
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if ((((uintptr_t)it.data | (uintptr_t)it.out) & 15) == 0) {
        const long long n4 = total >> 2;
        const float4* s = (const float4*)it.data; float4* d = (float4*)it.out;
        for (long long q = i; q < n4; q += stride) { float4 v = s[q]; v.x *= g; v.y *= g; v.z *= g; v.w *= g; d[q] = v; }
        for (long long q = (n4 << 2) + i; q < total; q += stride) it.out[q] = it.data[q] * g;
    } else {
        for (long long q = i; q < total; q += stride) it.out[q] = it.data[q] * g;
    }
}

// Internal (ss_internal.h): the measuring launches of ss_loudness_dev over n_items descriptors already in device memory,
// with k_loud_gate<true>: six launches, asynchronous on `stream`.
int loud_measure_enqueue(ss_ctx* c, const LoudItem* items, const int* prefix, int n_items, int total, double rate,
                         cudaStream_t stream) {
    const KCoef k = make_kcoef(rate);
    const dim3 scan_grid(8, n_items);
    k_kweight<1><<<(total + 127) / 128, 128, 0, stream>>>(items, prefix, n_items, k);
    k_kw_scan<<<scan_grid, 32, 0, stream>>>(items, 0);
    k_kweight<2><<<(total + 127) / 128, 128, 0, stream>>>(items, prefix, n_items, k);
    k_kw_scan<<<scan_grid, 32, 0, stream>>>(items, 1);
    k_kweight<3><<<(total + 127) / 128, 128, 0, stream>>>(items, prefix, n_items, k);
    k_loud_gate<true><<<n_items, kGateThreads, 0, stream>>>(items, n_items);
    CK(cudaGetLastError());
    c->launches += 6;
    return SS_OK;
}

// (stride_n, stride_c) describe a dense (N, C) or (C, N) block of N*C floats: k_loud_scale writes `out` as the N*C
// floats that follow it, so that is the only layout in which out[q] = gain * data[q] scales element (n, c) in place.
static bool dense_layout(int64_t N, int64_t C, int64_t sn, int64_t sc) {
    return (sc == 1 && (sn == C || N == 1)) || (sn == 1 && (sc == N || C == 1));
}

static int validate_loud(const ss_loud_item& it) {
    if (!it.data || !it.brk || !it.blk_lo || !it.blk_hi || !it.scratch || !it.result) return SS_ERR_INVALID;
    if (it.N <= 0 || it.C <= 0 || it.n_e <= 0 || it.n_blocks < 0 || it.rate <= 0) return SS_ERR_INVALID;
    if (it.C > 8) return SS_ERR_UNSUPPORTED;
    if (it.out && !dense_layout(it.N, it.C, it.stride_n, it.stride_c)) return SS_ERR_INVALID;   // measuring: any strides
    return SS_OK;
}

LoudItem to_item(const ss_loud_item& a) {
    LoudItem it;
    memset(&it, 0, sizeof(it));
    it.data = a.data; it.out = a.out; it.brk = a.brk; it.blk_lo = a.blk_lo; it.blk_hi = a.blk_hi;
    it.E = a.scratch; it.result = a.result;
    it.stride_n = a.stride_n; it.stride_c = a.stride_c;
    it.N = a.N; it.C = a.C; it.n_e = a.n_e; it.n_blocks = a.n_blocks;
    it.inv_norm = 1.0 / (a.block_size * a.rate);
    it.target = a.target_lufs;
    return it;
}

// all items must share one sample rate (one set of filter coefficients per launch)
extern "C" int ss_loudness_dev(ss_ctx* c, const ss_loud_item* items, int n_items, void* stream_) {
    if (!c || (!items && n_items > 0) || n_items < 0) return SS_ERR_INVALID;
    if (n_items == 0) return SS_OK;
    if (n_items > 65535) return SS_ERR_UNSUPPORTED;             // one gridDim.y row per item (k_kw_scan, k_loud_scale)
    CK(cudaSetDevice(c->device));
    cudaStream_t stream = (cudaStream_t)stream_;
    for (int i = 0; i < n_items; ++i) {
        int st = validate_loud(items[i]); if (st) return st;
        if (items[i].rate != items[0].rate) return SS_ERR_INVALID;
    }
    const size_t off_p = align_up(sizeof(LoudItem) * n_items, 16);
    const size_t bytes = off_p + align_up(sizeof(int) * (n_items + 1), 16);
    int slot; char *hblk, *dblk;
    { int st = ring_acquire(c, bytes, stream, &slot, &hblk, &dblk); if (st) return st; }
    LoudItem* h = (LoudItem*)c->h_desc[slot];
    int* hp = (int*)(c->h_desc[slot] + off_p);
    int tot = 0; bool any_out = false;
    for (int i = 0; i < n_items; ++i) {
        h[i] = to_item(items[i]);
        hp[i] = tot; tot += h[i].C * h[i].n_e;
        any_out = any_out || h[i].out != nullptr;
    }
    hp[n_items] = tot;
    CK(cudaMemcpyAsync(c->d_desc[slot], c->h_desc[slot], bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaEventRecord(c->desc_ev[slot], stream));
    const LoudItem* d = (const LoudItem*)c->d_desc[slot];
    const int* dp = (const int*)(c->d_desc[slot] + off_p);
    const KCoef k = make_kcoef(items[0].rate);
    const dim3 scan_grid(8, n_items);
    k_kweight<1><<<(tot + 127) / 128, 128, 0, stream>>>(d, dp, n_items, k);
    k_kw_scan<<<scan_grid, 32, 0, stream>>>(d, 0);
    k_kweight<2><<<(tot + 127) / 128, 128, 0, stream>>>(d, dp, n_items, k);
    k_kw_scan<<<scan_grid, 32, 0, stream>>>(d, 1);
    k_kweight<3><<<(tot + 127) / 128, 128, 0, stream>>>(d, dp, n_items, k);
    CK(cudaGetLastError());
    k_loud_gate<<<n_items, kGateThreads, 0, stream>>>(d, n_items);
    CK(cudaGetLastError());
    c->launches += 6;
    if (any_out) {
        dim3 grid(c->sm_count * 2, n_items);
        k_loud_scale<<<grid, 256, 0, stream>>>(d);
        CK(cudaGetLastError());
        c->launches += 1;
    }
    return ring_release(c, slot, stream);
}

// Internal (ss_internal.h): k_loud_scale alone, for stems that take the gain measured on another stem.
int loud_scale_dev(ss_ctx* c, const ScaleItem* items, int n_items, cudaStream_t stream) {
    if (n_items == 0) return SS_OK;
    const size_t bytes = sizeof(LoudItem) * n_items;
    int slot; char *hblk, *dblk;
    { int st = ring_acquire(c, bytes, stream, &slot, &hblk, &dblk); if (st) return st; }
    LoudItem* h = (LoudItem*)hblk;
    for (int i = 0; i < n_items; ++i) {
        memset(&h[i], 0, sizeof(LoudItem));
        h[i].data = items[i].data; h[i].out = items[i].data;
        h[i].result = const_cast<double*>(items[i].result);
        h[i].N = items[i].N; h[i].C = items[i].C;
    }
    CK(cudaMemcpyAsync(dblk, hblk, bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaEventRecord(c->desc_ev[slot], stream));
    k_loud_scale<<<dim3(c->sm_count * 2, n_items), 256, 0, stream>>>((const LoudItem*)dblk);
    CK(cudaGetLastError());
    c->launches += 1;
    return ring_release(c, slot, stream);
}

// Every stem with a target shares one sample rate (ss_loudness_dev runs one set of filter coefficients per call),
// checked against the first entry that has a target, so that the answer does not depend on how a caller groups stems.
// The `!(x > 0)` tests refuse NaN.
int check_post_lufs(const ss_post_lufs* post, int n) {
    const ss_post_lufs* first = nullptr;
    for (int i = 0; i < n; ++i) {
        const ss_post_lufs& q = post[i];
        if (!q.brk) continue;
        if (!q.blk_lo || !q.blk_hi || q.n_e <= 0 || q.n_blocks < 0 || !(q.rate > 0) || !(q.block_size > 0))
            return SS_ERR_INVALID;
        if (!first) first = &q;
        else if (q.rate != first->rate) return SS_ERR_INVALID;
    }
    return SS_OK;
}

// A table set: brk, then blk_lo at lo_at(q), then blk_hi at hi_at(q), each 256-aligned.  Stems of one clip length
// share the caller's host arrays (the normal case): their set is copied once.
static size_t lo_at(const ss_post_lufs& q) { return align_up(4 * (size_t)(q.n_e + 1), 256); }
static size_t hi_at(const ss_post_lufs& q) { return lo_at(q) + align_up(4 * (size_t)q.n_blocks + 4, 256); }

GatingTables gating_tables(const ss_post_lufs* post, int n) {
    GatingTables T;
    T.at.assign(n, 0);
    std::vector<int> sets;                               // the first entry of each distinct set
    for (int i = 0; i < n; ++i) {
        const ss_post_lufs& q = post[i];
        if (!q.brk) continue;
        const auto k = std::find_if(sets.begin(), sets.end(), [&](int j) {
            const ss_post_lufs& p = post[j];
            return p.brk == q.brk && p.blk_lo == q.blk_lo && p.blk_hi == q.blk_hi && p.n_e == q.n_e &&
                   p.n_blocks == q.n_blocks;
        });
        if (k != sets.end()) { T.at[i] = T.at[*k]; continue; }
        sets.push_back(i);
        const size_t off = T.bytes.size(), nb = 4 * (size_t)q.n_blocks;
        T.at[i] = off;
        T.bytes.resize(off + hi_at(q) + align_up(nb + 4, 256));
        memcpy(&T.bytes[off], q.brk, 4 * (size_t)(q.n_e + 1));
        if (nb) { memcpy(&T.bytes[off + lo_at(q)], q.blk_lo, nb); memcpy(&T.bytes[off + hi_at(q)], q.blk_hi, nb); }
    }
    return T;
}

ss_loud_item loud_item(const ss_post_lufs& q, const char* tab, const float* data, float* out, int32_t N, int32_t C,
                       double* scratch, double* result) {
    ss_loud_item it;
    memset(&it, 0, sizeof(it));
    it.data = data; it.out = out;
    it.brk = (const int32_t*)tab;
    it.blk_lo = (const int32_t*)(tab + lo_at(q)); it.blk_hi = (const int32_t*)(tab + hi_at(q));
    it.scratch = scratch; it.result = result;
    it.stride_n = 1; it.stride_c = N; it.N = N; it.C = C; it.n_e = q.n_e; it.n_blocks = q.n_blocks;
    it.rate = q.rate; it.block_size = q.block_size; it.target_lufs = q.target_lufs;
    return it;
}

// Single stem, host arrays (the drop-in lufs_norm): data / out hold N*C floats in the caller's layout, which is copied
// to the device as one block, so the strides must describe a dense layout even when only measuring.
extern "C" int ss_lufs_norm_host(ss_ctx* c, const float* data, float* out, int32_t N, int32_t C,
                                 int64_t stride_n, int64_t stride_c, double rate, double block_size,
                                 double target_lufs, const int32_t* brk, int32_t n_e, const int32_t* blk_lo,
                                 const int32_t* blk_hi, int32_t n_blocks, double* loudness, double* gain) {
    const ss_post_lufs q = {brk, blk_lo, blk_hi, n_e, n_blocks, rate, block_size, target_lufs, nullptr};
    if (!c || !data || !brk || N <= 0 || C <= 0 || check_post_lufs(&q, 1)) return SS_ERR_INVALID;
    if (!dense_layout(N, C, stride_n, stride_c)) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    // one block in the first input slot: the stem, its gating tables, the loudness scratch and the two result doubles
    const GatingTables tabs = gating_tables(&q, 1);
    const size_t nel = (size_t)N * C;
    const size_t o_tab = align_up(nel * 4, 256), o_scr = o_tab + tabs.bytes.size();
    const size_t o_res = o_scr + loud_scratch_bytes(q, C), total = o_res + 256;
    ss_ctx::Slot& sl = c->slot[0];
    CK(cudaStreamSynchronize(c->s_cmp));
    { const int rc = ensure(&sl.d_in, &sl.in_cap, total); if (rc) return rc; }
    char* base = sl.d_in;
    cudaStream_t st = c->s_cmp;
    CK(cudaMemcpyAsync(base, data, nel * 4, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(base + o_tab, tabs.bytes.data(), tabs.bytes.size(), cudaMemcpyHostToDevice, st));
    // scaled in place on the device; the copy keeps the caller's (dense) layout
    ss_loud_item it = loud_item(q, base + o_tab, (const float*)base, out ? (float*)base : nullptr, N, C,
                                (double*)(base + o_scr), (double*)(base + o_res));
    it.stride_n = stride_n; it.stride_c = stride_c;
    int rc = ss_loudness_dev(c, &it, 1, (void*)st);
    if (rc) return rc;
    double res[2];
    CK(cudaMemcpyAsync(res, base + o_res, sizeof(res), cudaMemcpyDeviceToHost, st));
    if (out) CK(cudaMemcpyAsync(out, base, nel * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (loudness) *loudness = res[0];
    if (gain) *gain = res[1];
    return SS_OK;
}
