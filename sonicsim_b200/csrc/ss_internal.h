// sonicsim_b200 :: ss_internal.h - host-side state shared by the translation units of the library.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>

#include "../../include/sonicsim_b200.h"

struct ss_ctx {
    int device = 0;
    int sm_count = 132;                      // H100 SXM; ss_create reads the device's own count
    int64_t chunk_bytes = 32ll << 20;        // device path: launch granularity; the spectra k_prepare writes for k_render
                                             // stay in the H100's 50 MB L2 (bench.py on H100: 16-32 MB equal, 40 MB -3 %,
                                             // 96 MB -9 %)
    int64_t chunk_bytes_host = 28ll << 20;   // host path: copy/compute/copy pipeline granularity (PCIe-bound)
    // scratch for spectra
    // kAux scratch buffers: consecutive chunks of ss_render_dev rotate through them (and through as many
    // internal streams) so that chunk i+1's descriptor copy + k_prepare overlap chunk i's k_render tail
#ifndef SS_AUX_STREAMS
#define SS_AUX_STREAMS 3
#endif
    static const int kAux = SS_AUX_STREAMS;
    char* d_scratch[kAux] = {}; size_t scratch_cap[kAux] = {};
    cudaStream_t s_aux[kAux] = {};
    cudaEvent_t ev_fork = nullptr, ev_join[kAux] = {};
    // descriptor ring (pinned host + device).  Any stream may reuse a slot (ring_acquire orders the reuse after the
    // slot's previous readers); kRing is a multiple of kAux so that ss_render_dev's forked chunks reuse each slot on
    // the stream that last used it, where that ordering costs nothing
    static const int kRing = 2 * SS_AUX_STREAMS;
    char* h_desc[kRing] = {};
    char* d_desc[kRing] = {};
    size_t desc_cap[kRing] = {};
    cudaEvent_t desc_ev[kRing] = {};     // behind the slot's host->device copy: the pinned block may be refilled
    cudaEvent_t desc_done[kRing] = {};   // behind the last launch that reads the slot's device block
    int ring_pos = 0;
    // host path
    cudaStream_t s_in = nullptr, s_cmp = nullptr, s_out = nullptr;
    struct Slot { char* d_in = nullptr; size_t in_cap = 0; char* d_out = nullptr; size_t out_cap = 0;
                  cudaEvent_t ev_in = nullptr, ev_done = nullptr, ev_free = nullptr, ev_rend = nullptr; } slot[4];
    // loudness post-processing of the host path: pinned block (results | gating tables) and its device twin
    char* h_post = nullptr; char* d_post = nullptr; size_t h_post_cap = 0;
    static const int kSlots = 4;   // H2D may run up to 3 chunks ahead of the D2H that frees a slot
    int64_t launches = 0;
    bool single_stream = false;   // experiment knob (SS_SINGLE_STREAM=1): no chunk overlap
    bool no_fast = false;         // experiment knob (SS_NO_FAST=1): never pick the all-aligned kernel variant
    bool no_graph = false;        // experiment knob (SS_NO_GRAPH=1): plans enqueue their launches instead of a CUDA graph
    // optional per-kernel timing (CUDA events on the launching stream)
    bool profiling = false;
    struct Prof { cudaEvent_t e0, e1, e2; int chunk; };   // chunk = position of the launch pair inside its render call
    int prof_chunk = 0;
    std::vector<Prof> prof;
};

extern thread_local int g_last_cuda;
#define CK(expr) do { cudaError_t e_ = (expr); if (e_ != cudaSuccess) { g_last_cuda = (int)e_; \
    return e_ == cudaErrorMemoryAllocation ? SS_ERR_NOMEM : SS_ERR_CUDA; } } while (0)


inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Grow-on-demand buffers of a context.  Growing waits for the whole device first: the old buffer may still be read by
// work on any stream.  ensure: the device buffer *p of *cap bytes to at least `need` (need + need / 4, in whole MB, so
// that slowly growing calls reallocate rarely).  ensure_pair: a pinned host block *h and its device twin *d, *cap bytes
// each, to at least `need` (twice `need`, in whole 4 KB pages).
inline int ensure(char** p, size_t* cap, size_t need) {
    if (need <= *cap) return SS_OK;
    CK(cudaDeviceSynchronize());
    if (*p) CK(cudaFree(*p));
    *p = nullptr; *cap = 0;
    const size_t grown = align_up(need + need / 4, 1 << 20);
    CK(cudaMalloc((void**)p, grown));
    *cap = grown;
    return SS_OK;
}
inline int ensure_pair(char** h, char** d, size_t* cap, size_t need) {
    if (need <= *cap) return SS_OK;
    CK(cudaDeviceSynchronize());
    if (*h) CK(cudaFreeHost(*h));
    if (*d) CK(cudaFree(*d));
    *h = nullptr; *d = nullptr; *cap = 0;
    const size_t grown = align_up(need * 2, 4096);
    CK(cudaHostAlloc((void**)h, grown, cudaHostAllocDefault));
    CK(cudaMalloc((void**)d, grown));
    *cap = grown;
    return SS_OK;
}

// data[i] *= (float)result[1] over the N * C floats of each item, with k_loud_scale's arithmetic: a stem that takes the
// linear gain another stem's loudness measurement left in `result` (ss_render_host_ex: the direct-path stem takes its
// reverberant stem's gain, so that target and mixture stay consistent).  Device pointers, asynchronous on `stream`.
struct ScaleItem { float* data; const double* result; int32_t N, C; };
int loud_scale_dev(ss_ctx* c, const ScaleItem* items, int n_items, cudaStream_t stream);

// Loudness targets of n stems (ss_render_host_ex, ss_pool_loudness).  check_post_lufs: the checks of ss_post_lufs in
// include/sonicsim_b200.h, SS_OK or SS_ERR_INVALID.  gating_tables: every distinct (brk, blk_lo, blk_hi, n_e, n_blocks)
// of the entries with a target once, in one host block for one upload; entry i's set at bytes[at[i]].
int check_post_lufs(const ss_post_lufs* post, int n);
struct GatingTables { std::vector<char> bytes; std::vector<size_t> at; };
GatingTables gating_tables(const ss_post_lufs* post, int n);
// The item that measures entry q's (C, N) stem at `data`, with its set of gating_tables at `tab` on the device;
// out = data normalises the stem in place, NULL measures only.  `scratch`: loud_scratch_bytes(q, C).
ss_loud_item loud_item(const ss_post_lufs& q, const char* tab, const float* data, float* out, int32_t N, int32_t C,
                       double* scratch, double* result);
// Loudness slots of plans (ss_stream_lufs): the device descriptor of item `a` (target_dev left null), and the measuring
// launches of ss_loudness_dev - k_kweight, k_kw_scan, k_loud_gate<true>, six launches - over n_items descriptors already
// in device memory, `prefix` their n_items + 1 work-item offsets (C * n_e each), all at one `rate`.
namespace ss { struct LoudItem; }
ss::LoudItem to_item(const ss_loud_item& a);
int loud_measure_enqueue(ss_ctx* c, const ss::LoudItem* items, const int* prefix, int n_items, int total, double rate,
                         cudaStream_t stream);
inline size_t loud_scratch_bytes(const ss_post_lufs& q, int32_t C) {
    return align_up(8 * (size_t)SS_LOUD_SCRATCH_DOUBLES * C * q.n_e, 256);
}

// One mixture of the dataloader's arithmetic (ss_mix.cu), as ss_mix_dev and plans with mixtures describe it on the
// device.  A stem is Cf rows of E floats at row stride T (Cf = 1: the stem's E floats as they are; Cf = C under
// SS_MIX_MONO: its (C, T) channels, folded to their mean at every element).
constexpr int kMixBlocks = 64;        // partial sums per mixture
constexpr int kMixStems = 8;          // at most 8 speakers and 8 noise stems per mixture
struct MixItem {
    const float* spk[kMixStems];     // speaker stems; speaker 0 is the reference
    const float* noise[kMixStems];   // noise stems
    const float* sirs;                // (S - 1) dB
    const float* snr;                 // dB, read by k_mix_write at every launch
    float* mix;                       // (E)
    float* spk_out;                   // (S, E) scaled speakers (may alias the speakers), or null
    float* rms_out;                   // (S) compute_mch_rms_dB of every speaker stem, or null
    double* scratch;                  // ss_mix_scratch_doubles(): kMixBlocks * (S + 2) partial sums, then the gains
    long long E, T;
    int S, M, Cf;
    int delay;                        // overlap_audio shift of the summed noise in elements (0 = none)
    float snr_val;                    // ss_mix_dev: the item's SNR, which `snr` points at in the uploaded descriptor
    // dereverberation targets (ss_plan_create_target), null elsewhere: dir[s] is speaker s's direct-path stem, laid out
    // as spk[s]; dir_out (S, E) receives each one folded and scaled by its speaker's gain, as spk_out does
    const float* dir[kMixStems];
    float* dir_out;
};
// The four mixture kernels over the n descriptors at `d` (device memory), asynchronous on `stream`; `direct`: some
// descriptor has a dir_out (k_mix_write<true>).
int mix_enqueue(ss_ctx* c, const MixItem* d, int n, cudaStream_t stream, bool direct = false);

// One level table of a pool candidate (ss_pool_levels): from the (C, N) stem y, q[0] = 0 and q[n + 1] = q[n] + e[n] in
// float64, e[n] the square of the mixture kernels' channel fold at n (mono) or the float64 sum of the C channels' squares.
struct LevelItem { const float* y; double* q; long long N; int C; int pad; };
// k_levels over the n descriptors at `d` (device memory), one CTA per table, asynchronous on `stream`.
int levels_enqueue(ss_ctx* c, const LevelItem* d, int n, bool mono, cudaStream_t stream);

// Take the next slot of the descriptor ring (pinned host block + its device twin), grown to `bytes`, for work on
// `stream`.  Blocks the host until the slot's previous host->device copy has completed (the pinned block is free), and
// makes `stream` wait for the slot's previous readers, whatever stream they ran on (the device block is free; a no-op
// wait when they ran on `stream`).  The caller fills `*h`, copies it to `*d` on `stream`, records c->desc_ev[*slot]
// right after the copy and c->desc_done[*slot] (ring_release) after the last launch that reads the slot.
inline int ring_acquire(ss_ctx* c, size_t bytes, cudaStream_t stream, int* slot_out, char** h, char** d) {
    const int slot = c->ring_pos; c->ring_pos = (c->ring_pos + 1) % ss_ctx::kRing;
    CK(cudaEventSynchronize(c->desc_ev[slot]));
    CK(cudaStreamWaitEvent(stream, c->desc_done[slot], 0));
    { const int st = ensure_pair(&c->h_desc[slot], &c->d_desc[slot], &c->desc_cap[slot], bytes); if (st) return st; }
    *slot_out = slot; *h = c->h_desc[slot]; *d = c->d_desc[slot];
    return SS_OK;
}
// Mark the end of the launches on `stream` that read ring slot `slot`.
inline int ring_release(ss_ctx* c, int slot, cudaStream_t stream) {
    CK(cudaEventRecord(c->desc_done[slot], stream));
    return SS_OK;
}
