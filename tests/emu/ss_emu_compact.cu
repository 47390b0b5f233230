// tests/emu/ss_emu_compact.cu - 16-bit dry pools (ss_dry_pool_create_i16) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE: runs what k_draw<true> and k_stage<true> run for a 16-bit dry pick - the sparse-table lookup
// (sparse_level, draw_silent_i16), the picked signal behind a pool's pointer array (speaker_signal_i16), the head of
// k_stage (stage_head) over a 16-bit pool's int16 signal table and the int16 -> float32 staging (i16x4_samples) - next to
// the float32 path over the same values.  Built with g++ (`-x c++`) by tests/test_compact_dry_pool.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// Q[s] of a 16-bit signal x from its sparse table q, for every s in ss[0..n)
void emu_sparse_levels(const double* q, const int16_t* x, const int* ss, int n, double* out) {
    for (int k = 0; k < n; ++k) out[k] = sparse_level(q, x, ss[k]);
}

// One draw as k_draw<true> makes it: S speakers, speaker k a float table (Q[k], D[k]) when x[k] is null, else a 16-bit
// dry signal x[k] with sparse table q[k] (D = len); M the draw's span.  Returns the start, *used the 1-based index of
// the kept try or 0.
int emu_draw_i16(const double* const* Q, const double* const* q, const int16_t* const* x, const double* D, int S,
                 int M, int len, const double* u, int tries, float threshold_db, int* used) {
    int s = 0;
    for (int t = 0; t < tries; ++t) {
        s = draw_start(u[t], M);
        bool silent = false;
        for (int k = 0; k < S; ++k)
            silent = silent || (x[k] ? draw_silent_i16(q[k], x[k], s, len, threshold_db)
                                     : draw_silent(Q[k], s, len, D[k], threshold_db));
        if (!silent) { *used = t + 1; return s; }
    }
    *used = 0;
    return s;
}

// A 16-bit pool's device pointer array as the library lays it out - n signal pointers, then n table pointers - read
// with dry pick v as k_draw<true> reads it: out[0] the index of the table speaker_table returns, out[1] the index of
// the signal speaker_signal_i16 returns (-1 if neither points into the pool)
void emu_speaker_i16(const int16_t* const* x, const double* const* q, int n, int v, int* out) {
    std::vector<const void*> ptrs(2 * (size_t)n);
    for (int i = 0; i < n; ++i) { ptrs[i] = x[i]; ptrs[n + i] = q[i]; }
    const double* const* levels = reinterpret_cast<const double* const*>(ptrs.data()) + n;
    const double* t = speaker_table(nullptr, nullptr, 0, levels, &v, n);
    const int16_t* sig = speaker_signal_i16(levels, &v, n);
    out[0] = out[1] = -1;
    for (int i = 0; i < n; ++i) {
        if (t == q[i]) out[0] = i;
        if (sig == x[i]) out[1] = i;
    }
}

// The head of k_stage for a dry-picked slot of a device pool (one candidate of N samples, P positions, bounds, K
// partitions) at window [ws, ws + wl), with dry pick dv into a pool of n_dry copies of one signal: once over a float32
// pool of the values d (k_stage<false>: whole float4s [x0, x1) copied) and once over a 16-bit pool of their int16 k
// (k_stage<true>: whole groups of 4 int16 converted by i16x4_samples), both arenas zero-padded to 64 bytes as the
// library pads them.  out_f / out_i receive the staged samples (x1 - x0 of each).  info receives [0..1] x0, x1 of the
// float pool, [2..3] of the 16-bit pool, [4..5] the error bits, [6] 1 if both views are the same, [7] 1 if the 16-bit
// staging read only inside the signal's padded arena span.
void emu_stage_i16(const int32_t* bounds, int N, int P, int C, int K, int ws, int wl, const float* d, const int16_t* k16,
                   int Nd, int n_dry, int dv, float* out_f, float* out_i, int* info) {
    PoolEntry e;
    memset(&e, 0, sizeof(e));
    e.bounds = P > 1 ? bounds : nullptr; e.N = N; e.P = P;
    const size_t padf = ((size_t)Nd * 4 + 63) / 64 * 16, padi = ((size_t)Nd * 2 + 63) / 64 * 32;   // samples
    std::vector<float> af(padf, 0.0f);
    std::vector<int16_t> ai(padi, 0);
    memcpy(af.data(), d, sizeof(float) * (size_t)Nd);
    memcpy(ai.data(), k16, sizeof(int16_t) * (size_t)Nd);
    std::vector<const float*> tf((size_t)n_dry, af.data());
    std::vector<const int16_t*> ti((size_t)n_dry, ai.data());
    StageView vf, vi;
    const float *sf = nullptr, *si = nullptr;
    int fx0, fx1, ix0, ix1;
    info[4] = (int)stage_head(&e, 1, 0, nullptr, K, nullptr, nullptr, ws, wl, C, false, tf.data(), dv, n_dry, vf, sf, fx0,
                              fx1);
    info[5] = (int)stage_head(&e, 1, 0, nullptr, K, nullptr, nullptr, ws, wl, C, false,
                              reinterpret_cast<const float* const*>(ti.data()), dv, n_dry, vi, si, ix0, ix1);
    info[0] = fx0; info[1] = fx1; info[2] = ix0; info[3] = ix1;
    info[6] = memcmp(&vf, &vi, sizeof(StageView)) == 0;
    info[7] = ix0 >= 0 && (size_t)ix1 <= padi && (ix0 & 3) == 0 && (ix1 & 3) == 0;
    for (int n = fx0; n < fx1; n += 4) memcpy(out_f + (n - fx0), sf + n, sizeof(float4));
    const short4* xs16 = reinterpret_cast<const short4*>(reinterpret_cast<const int16_t*>(si) + ix0);
    for (int g = 0; g < (ix1 - ix0) >> 2; ++g) {
        const float4 v = i16x4_samples(xs16[g]);
        memcpy(out_i + 4 * g, &v, sizeof(float4));
    }
}

}  // extern "C"
