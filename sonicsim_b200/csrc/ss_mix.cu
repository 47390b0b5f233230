// sonicsim_b200 :: ss_mix.cu - mixture assembly of the training dataloader
// (separation/look2hear/datas/movingdatamodule.py:29-32,105-124): active-energy (RMS dB) of the
// reference speaker, SIR gains of the interferers (clamped to +40 dB), sum, SNR gain of the summed
// noise, sum.  Three streaming passes over stems that are already in HBM + one tiny gain kernel;
// per-block partial sums are combined in a fixed order, so results are run-to-run deterministic.
#include <math.h>
#include <stddef.h>
#include <string.h>

#include "ss_internal.h"

namespace {

constexpr int kMaxStems = kMixStems;
constexpr uint64_t kMaxE = UINT64_MAX / 4 / kMaxStems;   // so that the byte size of any (S, E) or (M, E) block fits

__device__ __forceinline__ double block_sum(double v, double* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) sh[w] = v;
    __syncthreads();
    double r = 0;
    if (threadIdx.x == 0) for (int i = 0; i < (int)(blockDim.x >> 5); ++i) r += sh[i];
    return r;          // valid in thread 0
}

// element e of a stem: its own value (Cf = 1), or the mean of its Cf channel rows at e - a float32 sum in channel order
// 0..Cf-1, every add rounded on its own, then an IEEE division by Cf.  fold4 gives the same bits four elements at a time.
__device__ __forceinline__ float fold(const MixItem& it, const float* p, long long e) {
    float v = p[e];
    if (it.Cf == 1) return v;
    for (int c = 1; c < it.Cf; ++c) v = __fadd_rn(v, p[(long long)c * it.T + e]);
    return __fdiv_rn(v, (float)it.Cf);
}
__device__ __forceinline__ float4 fold4(const MixItem& it, const float* p, long long q) {
    float4 v = ((const float4*)p)[q];
    if (it.Cf == 1) return v;
    for (int c = 1; c < it.Cf; ++c) {
        const float4 a = ((const float4*)(p + (long long)c * it.T))[q];
        v.x = __fadd_rn(v.x, a.x); v.y = __fadd_rn(v.y, a.y); v.z = __fadd_rn(v.z, a.z); v.w = __fadd_rn(v.w, a.w);
    }
    const float C = (float)it.Cf;
    v.x = __fdiv_rn(v.x, C); v.y = __fdiv_rn(v.y, C); v.z = __fdiv_rn(v.z, C); v.w = __fdiv_rn(v.w, C);
    return v;
}

// summed noise stems at element e; with delay D > 0 the enhancement dataloader's overlap_audio
// (enhancement/look2hear/datas/movingdatamodule.py:34-48) on top: (s[e-D] + s[e+D]) + s[e], zeros outside [0, E)
__device__ __forceinline__ float noise_sum(const MixItem& it, long long e) {
    float n = 0.f;
    for (int m = 0; m < it.M; ++m) n += fold(it, it.noise[m], e);
    return n;
}
__device__ __forceinline__ float noise_at(const MixItem& it, long long e) {
    const float n = noise_sum(it, e);
    if (it.delay <= 0) return n;
    const float f = e >= it.delay ? noise_sum(it, e - it.delay) : 0.f;
    const float b = e + it.delay < it.E ? noise_sum(it, e + it.delay) : 0.f;
    return __fadd_rn(__fadd_rn(f, b), n);
}

// 16-byte path of the three streaming passes: element count (and channel stride) a multiple of 4, every row 16-byte
// aligned, no overlap_audio shift (whose +-D neighbours need not be aligned)
__device__ __forceinline__ bool mix_vec_ok(const MixItem& it) {
    if (it.delay > 0 || (it.E & 3) != 0 || (it.Cf > 1 && (it.T & 3) != 0)) return false;
    uintptr_t a = (uintptr_t)it.mix | (uintptr_t)it.spk_out;
    for (int s = 0; s < it.S; ++s) a |= (uintptr_t)it.spk[s];
    for (int m = 0; m < it.M; ++m) a |= (uintptr_t)it.noise[m];
    return (a & 15) == 0;
}
__device__ __forceinline__ float4 noise_sum4(const MixItem& it, long long q) {
    float4 n = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int m = 0; m < it.M; ++m) {
        const float4 v = fold4(it, it.noise[m], q);
        n.x += v.x; n.y += v.y; n.z += v.z; n.w += v.w;
    }
    return n;
}

// pass 1: sum of squares of every speaker stem and of the summed noise
__global__ void __launch_bounds__(256) k_mix_energy(const MixItem* __restrict__ items) {
    __shared__ double sh[8];
    const MixItem& it = items[blockIdx.y];
    double acc[kMaxStems + 1];
#pragma unroll
    for (int i = 0; i <= kMaxStems; ++i) acc[i] = 0;
    if (mix_vec_ok(it)) {
        for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < (it.E >> 2); q += (long long)gridDim.x * blockDim.x) {
#pragma unroll
            for (int s = 0; s < kMaxStems; ++s) if (s < it.S) {
                const float4 v = fold4(it, it.spk[s], q);
                acc[s] += (double)(v.x * v.x) + (double)(v.y * v.y) + (double)(v.z * v.z) + (double)(v.w * v.w);
            }
            const float4 n = noise_sum4(it, q);
            acc[kMaxStems] += (double)(n.x * n.x) + (double)(n.y * n.y) + (double)(n.z * n.z) + (double)(n.w * n.w);
        }
    } else
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < it.E; e += (long long)gridDim.x * blockDim.x) {
#pragma unroll
        for (int s = 0; s < kMaxStems; ++s) if (s < it.S) { float v = fold(it, it.spk[s], e); acc[s] += (double)(v * v); }
        const float n = noise_at(it, e);
        acc[kMaxStems] += (double)(n * n);
    }
#pragma unroll
    for (int s = 0; s <= kMaxStems; ++s) {
        if (s < it.S || s == kMaxStems) {
            double r = block_sum(acc[s], sh);
            if (threadIdx.x == 0) it.scratch[(long long)blockIdx.x * (kMaxStems + 2) + s] = r;
        }
    }
}

__device__ double rms_db(double sum_sq, long long count) {
    double ms = sum_sq / (double)count;               // torch.mean(x ** 2)
    if (ms < 1e-20) ms = 1e-20;                       // max(1e-20, .)   movingdatamodule.py:31
    return 10.0 * log10(ms);
}

// gains of the interferers: gain_i = min(E(spk0) - E(spk_i) - sir_i, 40) dB   (:108-113); the speakers' E to rms_out
__global__ void k_mix_gain(const MixItem* __restrict__ items, int n) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const MixItem& it = items[i];
    double tot[kMaxStems + 1];
    for (int s = 0; s <= kMaxStems; ++s) tot[s] = 0;
    for (int b = 0; b < kMixBlocks; ++b)
        for (int s = 0; s <= kMaxStems; ++s) if (s < it.S || s == kMaxStems) tot[s] += it.scratch[(long long)b * (kMaxStems + 2) + s];
    double* g = it.scratch + (long long)kMixBlocks * (kMaxStems + 2);
    const double target = rms_db(tot[0], it.E);
    g[0] = 1.0;
    for (int s = 1; s < it.S; ++s) {
        double gain = target - rms_db(tot[s], it.E) - (double)it.sirs[s - 1];
        if (gain > 40.0) gain = 40.0;
        g[s] = pow(10.0, gain / 20.0);
    }
    // rms_db's value again with a product of its own (__dmul_rn), so that the gains above keep their contraction
    if (it.rms_out)
        for (int s = 0; s < it.S; ++s) {
            double ms = tot[s] / (double)it.E;
            if (ms < 1e-20) ms = 1e-20;
            it.rms_out[s] = (float)__dmul_rn(10.0, log10(ms));
        }
    g[kMaxStems] = rms_db(tot[kMaxStems], it.E);      // noise energy (dB), consumed by k_mix_write
}

// pass 2: energy of all_speech = sum_i g_i spk_i
__global__ void __launch_bounds__(256) k_mix_speech_energy(const MixItem* __restrict__ items) {
    __shared__ double sh[8];
    const MixItem& it = items[blockIdx.y];
    const double* g = it.scratch + (long long)kMixBlocks * (kMaxStems + 2);
    float gf[kMaxStems];
#pragma unroll
    for (int s = 0; s < kMaxStems; ++s) gf[s] = s < it.S ? (float)g[s] : 0.f;
    double acc = 0;
    if (mix_vec_ok(it)) {
        for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < (it.E >> 2); q += (long long)gridDim.x * blockDim.x) {
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int s = 0; s < kMaxStems; ++s) if (s < it.S) {
                const float4 a = fold4(it, it.spk[s], q);
                v.x += a.x * gf[s]; v.y += a.y * gf[s]; v.z += a.z * gf[s]; v.w += a.w * gf[s];
            }
            acc += (double)(v.x * v.x) + (double)(v.y * v.y) + (double)(v.z * v.z) + (double)(v.w * v.w);
        }
    } else
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < it.E; e += (long long)gridDim.x * blockDim.x) {
        float v = 0.f;
#pragma unroll
        for (int s = 0; s < kMaxStems; ++s) if (s < it.S) v += fold(it, it.spk[s], e) * gf[s];
        acc += (double)(v * v);
    }
    double r = block_sum(acc, sh);
    if (threadIdx.x == 0) it.scratch[(long long)blockIdx.x * (kMaxStems + 2) + kMaxStems + 1] = r;
}

// The write pass's 16-byte test: mix_vec_ok, and with kDirect also a target's direct rows and dir_out.  The pass writes
// every element on its own, so either path gives the same bits and the choice may differ from the energy passes'.
template <bool kDirect>
__device__ __forceinline__ bool write_vec_ok(const MixItem& it) {
    if (!mix_vec_ok(it)) return false;
    if (!kDirect || !it.dir_out) return true;
    uintptr_t a = (uintptr_t)it.dir_out;
    for (int s = 0; s < it.S; ++s) a |= (uintptr_t)it.dir[s];
    return (a & 15) == 0;
}

// pass 3: noise gain (:118-121), mixture and scaled speakers (:123-124); with kDirect, a mixture with dir_out also
// writes each speaker's folded direct-path stem times the speaker's gain gf[s], with the multiply of spk_out
template <bool kDirect>
__global__ void __launch_bounds__(256) k_mix_write(const MixItem* __restrict__ items) {
    const MixItem& it = items[blockIdx.y];
    const double* g = it.scratch + (long long)kMixBlocks * (kMaxStems + 2);
    double tot = 0;
    for (int b = 0; b < kMixBlocks; ++b) tot += it.scratch[(long long)b * (kMaxStems + 2) + kMaxStems + 1];
    double gain = rms_db(tot, it.E) - g[kMaxStems] - (double)*it.snr;
    if (gain > 40.0) gain = 40.0;
    const float gn = (float)pow(10.0, gain / 20.0);
    float gf[kMaxStems];
#pragma unroll
    for (int s = 0; s < kMaxStems; ++s) gf[s] = s < it.S ? (float)g[s] : 0.f;
    if (write_vec_ok<kDirect>(it)) {
        for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < (it.E >> 2); q += (long long)gridDim.x * blockDim.x) {
            float4 sp = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
            for (int s = 0; s < kMaxStems; ++s) if (s < it.S) {
                float4 v = fold4(it, it.spk[s], q);
                v.x = __fmul_rn(v.x, gf[s]); v.y = __fmul_rn(v.y, gf[s]); v.z = __fmul_rn(v.z, gf[s]); v.w = __fmul_rn(v.w, gf[s]);
                if (it.spk_out) ((float4*)(it.spk_out + (long long)s * it.E))[q] = v;
                sp.x += v.x; sp.y += v.y; sp.z += v.z; sp.w += v.w;
                if (kDirect && it.dir_out) {
                    float4 d = fold4(it, it.dir[s], q);
                    d.x = __fmul_rn(d.x, gf[s]); d.y = __fmul_rn(d.y, gf[s]); d.z = __fmul_rn(d.z, gf[s]); d.w = __fmul_rn(d.w, gf[s]);
                    ((float4*)(it.dir_out + (long long)s * it.E))[q] = d;
                }
            }
            const float4 n = noise_sum4(it, q);
            float4 o;
            o.x = __fadd_rn(sp.x, __fmul_rn(n.x, gn)); o.y = __fadd_rn(sp.y, __fmul_rn(n.y, gn));
            o.z = __fadd_rn(sp.z, __fmul_rn(n.z, gn)); o.w = __fadd_rn(sp.w, __fmul_rn(n.w, gn));
            ((float4*)it.mix)[q] = o;
        }
        return;
    }
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < it.E; e += (long long)gridDim.x * blockDim.x) {
        float sp = 0.f;
#pragma unroll
        for (int s = 0; s < kMaxStems; ++s) if (s < it.S) {
            float v = __fmul_rn(fold(it, it.spk[s], e), gf[s]);               // products and sums rounded separately, as torch does
            if (it.spk_out) it.spk_out[(long long)s * it.E + e] = v;
            sp += v;
            if (kDirect && it.dir_out) it.dir_out[(long long)s * it.E + e] = __fmul_rn(fold(it, it.dir[s], e), gf[s]);
        }
        it.mix[e] = __fadd_rn(sp, __fmul_rn(noise_at(it, e), gn));
    }
}

// Level tables of pool candidates (ss_pool_levels): one CTA per table walks the stem in tiles of kLevelThreads *
// kLevelPer samples.  Each thread sums its kLevelPer consecutive terms in order, a warp shuffle scan and the warps'
// totals in warp order place them in the tile, and a carry runs from tile to tile, so the bits depend on N alone: not
// on the grouping, the launch or the run.  The mono term is fold() itself, the term k_mix_energy squares.
constexpr int kLevelThreads = 256, kLevelPer = 8;
__global__ void __launch_bounds__(kLevelThreads) k_levels(const LevelItem* __restrict__ items, int mono) {
    __shared__ double sh[kLevelThreads / 32];
    const LevelItem L = items[blockIdx.x];
    MixItem it;
    it.Cf = L.C; it.T = L.N;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) L.q[0] = 0.0;
    double carry = 0.0;
    for (long long base = 0; base < L.N; base += (long long)kLevelThreads * kLevelPer) {
        const long long n0 = base + (long long)threadIdx.x * kLevelPer;
        double run[kLevelPer];
        double acc = 0.0;
#pragma unroll
        for (int j = 0; j < kLevelPer; ++j) {
            const long long n = n0 + j;
            double e = 0.0;
            if (n < L.N) {
                if (mono) { const float v = fold(it, L.y, n); e = (double)(v * v); }
                else for (int c = 0; c < L.C; ++c) { const float v = L.y[(long long)c * L.N + n]; e += (double)(v * v); }
            }
            acc += e;
            run[j] = acc;
        }
        double incl = acc;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const double v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
        double excl = __shfl_up_sync(0xffffffffu, incl, 1);
        if (lane == 0) excl = 0.0;
        if (lane == 31) sh[warp] = incl;
        __syncthreads();
        double wpre = 0.0, tile = 0.0;
        for (int w = 0; w < kLevelThreads / 32; ++w) { if (w < warp) wpre += sh[w]; tile += sh[w]; }
        const double pre = carry + (wpre + excl);
#pragma unroll
        for (int j = 0; j < kLevelPer; ++j)
            if (n0 + j < L.N) L.q[n0 + j + 1] = pre + run[j];
        carry += tile;
        __syncthreads();                                  // sh is rewritten by the next tile
    }
}

// true when the byte ranges [a, a + na) and [b, b + nb) share a byte
bool ranges_meet(const void* a, size_t na, const void* b, size_t nb) {
    const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
    return na > 0 && nb > 0 && x < y + nb && y < x + na;
}

// The kernels read an item's inputs while other CTAs write its outputs, so every range an item writes (mix, scratch,
// a separate speakers_out) must meet no other range of the item; speakers_out may instead be exactly `speakers`.
bool mix_item_disjoint(const ss_mix_item& a) {
    const bool alias = a.speakers_out == a.speakers;
    struct R { const void* p; size_t n; bool written; } r[6] = {
        {a.speakers, 4 * (size_t)a.S * a.E, alias},
        {a.noises, 4 * (size_t)a.M * a.E, false},
        {a.sirs, 4 * (size_t)(a.S - 1), false},
        {a.mix, 4 * (size_t)a.E, true},
        {a.scratch, 8 * (size_t)(kMixBlocks * (kMaxStems + 2) + kMaxStems + 1), true},
        {alias ? nullptr : a.speakers_out, a.speakers_out && !alias ? 4 * (size_t)a.S * a.E : 0, true}};
    for (int i = 0; i < 6; ++i)
        for (int j = i + 1; j < 6; ++j)
            if ((r[i].written || r[j].written) && ranges_meet(r[i].p, r[i].n, r[j].p, r[j].n)) return false;
    return true;
}

}  // namespace

extern "C" int ss_mix_dev(ss_ctx* c, const ss_mix_item* items, int n_items, void* stream_) {
    if (!c || (!items && n_items > 0) || n_items < 0) return SS_ERR_INVALID;
    if (n_items == 0) return SS_OK;
    if (n_items > 65535) return SS_ERR_UNSUPPORTED;             // one gridDim.y row per item
    for (int i = 0; i < n_items; ++i) {
        const ss_mix_item& a = items[i];
        if (!a.speakers || !a.noises || !a.mix || !a.scratch || a.E <= 0 || a.S < 1 || a.M < 1) return SS_ERR_INVALID;
        if (a.S > kMaxStems || a.M > kMaxStems) return SS_ERR_UNSUPPORTED;
        if ((uint64_t)a.E > kMaxE) return SS_ERR_INVALID;
        if (a.S > 1 && !a.sirs) return SS_ERR_INVALID;
        if (a.noise_delay < 0) return SS_ERR_INVALID;
        if (!mix_item_disjoint(a)) return SS_ERR_INVALID;
    }
    CK(cudaSetDevice(c->device));
    cudaStream_t stream = (cudaStream_t)stream_;
    const size_t bytes = align_up(sizeof(MixItem) * n_items, 16);
    int slot; char *hblk, *dblk;
    { int st = ring_acquire(c, bytes, stream, &slot, &hblk, &dblk); if (st) return st; }
    MixItem* h = (MixItem*)c->h_desc[slot];
    for (int i = 0; i < n_items; ++i) {
        const ss_mix_item& a = items[i];
        MixItem m; memset(&m, 0, sizeof(m));
        for (int s = 0; s < a.S; ++s) m.spk[s] = a.speakers + (long long)s * a.E;
        for (int q = 0; q < a.M; ++q) m.noise[q] = a.noises + (long long)q * a.E;
        m.sirs = a.sirs; m.mix = a.mix; m.spk_out = a.speakers_out; m.scratch = a.scratch;
        m.E = a.E; m.T = a.E; m.S = a.S; m.M = a.M; m.Cf = 1; m.delay = a.noise_delay;
        m.snr_val = a.snr;
        m.snr = (const float*)(c->d_desc[slot] + sizeof(MixItem) * i + offsetof(MixItem, snr_val));
        h[i] = m;
    }
    CK(cudaMemcpyAsync(c->d_desc[slot], c->h_desc[slot], bytes, cudaMemcpyHostToDevice, stream));
    CK(cudaEventRecord(c->desc_ev[slot], stream));
    const int st = mix_enqueue(c, (const MixItem*)c->d_desc[slot], n_items, stream);   // k_mix_write reads the SNR here
    const int rs = ring_release(c, slot, stream);
    return st ? st : rs;
}

int mix_enqueue(ss_ctx* c, const MixItem* d, int n, cudaStream_t stream, bool direct) {
    dim3 grid(kMixBlocks, n);
    k_mix_energy<<<grid, 256, 0, stream>>>(d);
    k_mix_gain<<<(n + 63) / 64, 64, 0, stream>>>(d, n);
    k_mix_speech_energy<<<grid, 256, 0, stream>>>(d);
    if (direct) k_mix_write<true><<<grid, 256, 0, stream>>>(d);
    else k_mix_write<false><<<grid, 256, 0, stream>>>(d);
    CK(cudaGetLastError());
    c->launches += 4;
    return SS_OK;
}

int levels_enqueue(ss_ctx* c, const LevelItem* d, int n, bool mono, cudaStream_t stream) {
    k_levels<<<n, kLevelThreads, 0, stream>>>(d, mono ? 1 : 0);
    CK(cudaGetLastError());
    c->launches += 1;
    return SS_OK;
}

extern "C" int64_t ss_mix_scratch_doubles(void) { return (int64_t)kMixBlocks * (kMaxStems + 2) + kMaxStems + 1; }

extern "C" int ss_mix_host_ex(ss_ctx* c, const float* speakers, const float* noises, const float* sirs, float snr,
                              float* mix, float* speakers_out, int32_t S, int32_t M, int64_t E, int32_t noise_delay) {
    if (!c || !speakers || !noises || !mix || S < 1 || M < 1 || E <= 0 || noise_delay < 0) return SS_ERR_INVALID;
    if (S > kMaxStems || M > kMaxStems) return SS_ERR_UNSUPPORTED;       // ss_mix_dev's limits, before any upload
    if ((uint64_t)E > kMaxE || (S > 1 && !sirs)) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    const size_t o_spk = 0, o_noise = align_up(4 * (size_t)S * E, 256), o_mix = o_noise + align_up(4 * (size_t)M * E, 256);
    const size_t o_sir = o_mix + align_up(4 * (size_t)E, 256), o_scr = o_sir + 256;
    const size_t total = o_scr + align_up(8 * (size_t)ss_mix_scratch_doubles(), 256);
    ss_ctx::Slot& sl = c->slot[0];
    cudaStream_t st = c->s_cmp;
    CK(cudaStreamSynchronize(st));
    { const int rc = ensure(&sl.d_in, &sl.in_cap, total); if (rc) return rc; }
    char* b = sl.d_in;
    CK(cudaMemcpyAsync(b + o_spk, speakers, 4 * (size_t)S * E, cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(b + o_noise, noises, 4 * (size_t)M * E, cudaMemcpyHostToDevice, st));
    if (S > 1) CK(cudaMemcpyAsync(b + o_sir, sirs, 4 * (size_t)(S - 1), cudaMemcpyHostToDevice, st));
    ss_mix_item it; memset(&it, 0, sizeof(it));
    it.speakers = (const float*)(b + o_spk); it.noises = (const float*)(b + o_noise); it.sirs = (const float*)(b + o_sir);
    it.mix = (float*)(b + o_mix); it.speakers_out = speakers_out ? (float*)(b + o_spk) : nullptr;
    it.scratch = (double*)(b + o_scr); it.E = E; it.S = S; it.M = M; it.snr = snr; it.noise_delay = noise_delay;
    int rc = ss_mix_dev(c, &it, 1, (void*)st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(mix, b + o_mix, 4 * (size_t)E, cudaMemcpyDeviceToHost, st));
    if (speakers_out) CK(cudaMemcpyAsync(speakers_out, b + o_spk, 4 * (size_t)S * E, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SS_OK;
}

extern "C" int ss_mix_host(ss_ctx* c, const float* speakers, const float* noises, const float* sirs, float snr,
                           float* mix, float* speakers_out, int32_t S, int32_t M, int64_t E) {
    return ss_mix_host_ex(c, speakers, noises, sirs, snr, mix, speakers_out, S, M, E, 0);
}

// ---- overlap_audio (enhancement/look2hear/datas/movingdatamodule.py:34-48) as a stand-alone op
namespace {
__global__ void __launch_bounds__(256) k_overlap(const float* __restrict__ x, float* __restrict__ y, long long T, long long D) {
    const float* xr = x + (long long)blockIdx.y * T;
    float* yr = y + (long long)blockIdx.y * T;
    for (long long n = (long long)blockIdx.x * blockDim.x + threadIdx.x; n < T; n += (long long)gridDim.x * blockDim.x) {
        const float f = n >= D ? xr[n - D] : 0.f;
        const float b = n + D < T ? xr[n + D] : 0.f;
        yr[n] = __fadd_rn(__fadd_rn(f, b), xr[n]);
    }
}
}  // namespace

extern "C" int ss_overlap_dev(ss_ctx* c, const float* x, float* y, int32_t rows, int64_t T, int64_t delay, void* stream_) {
    if (!c || !x || !y || x == y || rows < 0 || T < 0 || delay < 0) return SS_ERR_INVALID;
    if (rows == 0 || T == 0) return SS_OK;
    if (rows > 65535) return SS_ERR_UNSUPPORTED;
    // k_overlap reads x[n +- D] that other threads may be writing when y overlaps x
    if ((uint64_t)T > UINT64_MAX / 4 / (uint64_t)rows) return SS_ERR_INVALID;
    const size_t bytes = 4 * (size_t)rows * (size_t)T;
    if (ranges_meet(x, bytes, y, bytes)) return SS_ERR_INVALID;
    CK(cudaSetDevice(c->device));
    long long nb = (T + 255) / 256;
    if (nb > 8ll * c->sm_count) nb = 8ll * c->sm_count;   // 8 waves of CTAs, grid-stride beyond that
    k_overlap<<<dim3((unsigned)nb, (unsigned)rows), 256, 0, (cudaStream_t)stream_>>>(x, y, T, delay);
    CK(cudaGetLastError());
    c->launches += 1;
    return SS_OK;
}

extern "C" int ss_overlap_host(ss_ctx* c, const float* x, float* y, int32_t rows, int64_t T, int64_t delay) {
    if (!c || !x || !y || rows < 0 || T < 0 || delay < 0) return SS_ERR_INVALID;
    if (rows == 0 || T == 0) return SS_OK;
    CK(cudaSetDevice(c->device));
    const size_t bytes = 4 * (size_t)rows * (size_t)T, o_y = align_up(bytes, 256), total = o_y + align_up(bytes, 256);
    ss_ctx::Slot& sl = c->slot[0];
    cudaStream_t st = c->s_cmp;
    CK(cudaStreamSynchronize(st));
    { const int rc = ensure(&sl.d_in, &sl.in_cap, total); if (rc) return rc; }
    char* b = sl.d_in;
    CK(cudaMemcpyAsync(b, x, bytes, cudaMemcpyHostToDevice, st));
    int rc = ss_overlap_dev(c, (const float*)b, (float*)(b + o_y), rows, T, delay, (void*)st);
    if (rc) return rc;
    CK(cudaMemcpyAsync(y, b + o_y, bytes, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return SS_OK;
}
