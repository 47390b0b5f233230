// sonicsim_b200 :: ss_loud.cuh - ITU-R BS.1770 loudness (K-weighting + gated mean square) as
// pyloudnorm 0.1.1 computes it for SonicSim_audio.lufs_norm (SonicSim_audio.py:68-81).
// Host/device per-thread code, shared with the CPU emulation in tests/emu.
#pragma once
#include "ss_core.cuh"
#include <math.h>

namespace ss {

// two RBJ biquads, a0-normalised: high shelf (+4 dB, Q = 1/sqrt 2, 1500 Hz), high pass (Q = 0.5, 38 Hz)
struct KCoef { double b0[2], b1[2], b2[2], a1[2], a2[2]; };

inline KCoef make_kcoef(double rate) {
    KCoef k;
    const double PI = 3.14159265358979323846;
    {   // high shelf
        double G = 4.0, Q = 1.0 / sqrt(2.0), fc = 1500.0;
        double A = pow(10.0, G / 40.0), w0 = 2.0 * PI * (fc / rate), alpha = sin(w0) / (2.0 * Q);
        double b0 = A * ((A + 1) + (A - 1) * cos(w0) + 2 * sqrt(A) * alpha);
        double b1 = -2 * A * ((A - 1) + (A + 1) * cos(w0));
        double b2 = A * ((A + 1) + (A - 1) * cos(w0) - 2 * sqrt(A) * alpha);
        double a0 = (A + 1) - (A - 1) * cos(w0) + 2 * sqrt(A) * alpha;
        double a1 = 2 * ((A - 1) - (A + 1) * cos(w0));
        double a2 = (A + 1) - (A - 1) * cos(w0) - 2 * sqrt(A) * alpha;
        k.b0[0] = b0 / a0; k.b1[0] = b1 / a0; k.b2[0] = b2 / a0; k.a1[0] = a1 / a0; k.a2[0] = a2 / a0;
    }
    {   // high pass
        double Q = 0.5, fc = 38.0;
        double w0 = 2.0 * PI * (fc / rate), alpha = sin(w0) / (2.0 * Q);
        double b0 = (1 + cos(w0)) / 2, b1 = -(1 + cos(w0)), b2 = (1 + cos(w0)) / 2;
        double a0 = 1 + alpha, a1 = -2 * cos(w0), a2 = 1 - alpha;
        k.b0[1] = b0 / a0; k.b1[1] = b1 / a0; k.b2[1] = b2 / a0; k.a1[1] = a1 / a0; k.a2[1] = a2 / a0;
    }
    return k;
}

// One stem to measure (and optionally normalise).  Element (n, c) is data[n * stride_n + c * stride_c].
struct LoudItem {
    const float* data;
    float* out;              // C*N contiguous floats scaled by the gain (may alias data); null = measure only
    const int* brk;          // n_e + 1 ascending sample indices: the gating blocks' distinct bounds
    const int* blk_lo;       // per gating block j: first elementary interval
    const int* blk_hi;       // per gating block j: one past its last elementary interval
    double* E;               // scratch, kLoudScratch * C * n_e doubles: [0, C n_e) interval energies (sum of squares of
                             // the K-weighted signal), then the per-interval filter states of the three passes below
    double* result;          // [0] integrated loudness (LUFS, -inf allowed), [1] linear gain applied
    long long stride_n, stride_c;
    int N, C, n_e, n_blocks;
    const double* target_dev;   // k_loud_gate<true> (loudness slots of plans): the target LUFS, read at every run;
                                // null elsewhere (in the bytes that were padding, so that the layout is unchanged)
    double inv_norm;         // 1 / (T_g * rate)
    double target;           // target LUFS (SonicSim_audio.py:77 `norm`)
};
static_assert(sizeof(LoudItem) == 112, "LoudItem layout");
constexpr int kLoudScratch = 20;   // doubles of scratch per (channel, elementary interval)

// ---- K-weighting of one channel, EXACT and parallel over the elementary intervals.
// pyloudnorm filters the whole channel with scipy.signal.lfilter (direct form II transposed, float64), stage by
// stage, storing each stage back into its float32 array.  The recursion is linear, so the state at the start of
// interval e is   S_e = M^len(e-1) S_(e-1) + F_(e-1),   F = state at the end of an interval filtered from rest,
// M = [[-a1, 1], [-a2, 0]].  Three passes, one thread per (channel, interval), each over its own samples only:
//   pass 1  stage 1 from rest                                  -> F1, and M1^len, M2^len by repeated squaring
//   scan 1  S1 of every interval from (M1^len, F1): a scan over affine maps, one warp per channel on the device
//   pass 2  stage 1 exact from S1, its float32 output through stage 2 from rest -> F2
//   scan 2  S2 likewise
//   pass 3  both stages exact; energy of the float32 output
// No warm-up approximation: the result differs from lfilter's only by float64 rounding of the state recurrence.
struct Mat2 { double a, b, c, d; };
SS_HD Mat2 mat_mul(const Mat2& x, const Mat2& y) {
    Mat2 r; r.a = x.a * y.a + x.b * y.c; r.b = x.a * y.b + x.b * y.d; r.c = x.c * y.a + x.d * y.c; r.d = x.c * y.b + x.d * y.d;
    return r;
}
SS_HD Mat2 mat_pow(Mat2 m, int n) {
    Mat2 r; r.a = 1; r.b = 0; r.c = 0; r.d = 1;
    while (n > 0) { if (n & 1) r = mat_mul(r, m); m = mat_mul(m, m); n >>= 1; }
    return r;
}
SS_HD Mat2 stage_matrix(const KCoef& k, int s) { Mat2 m; m.a = -k.a1[s]; m.b = 1.0; m.c = -k.a2[s]; m.d = 0.0; return m; }

// scratch slots of (channel c, interval e)
SS_HD double* loud_slot(const LoudItem& it, int which, int c, int e) {
    // which: 0 E(1) | 1 F1(2) | 2 S1(2) | 3 F2(2) | 4 M1(4) | 5 M2(4) | 6 S2(2)
    const long long ce = (long long)it.C * it.n_e, i = (long long)c * it.n_e + e;
    switch (which) {
        case 0: return it.E + i;
        case 1: return it.E + ce + 2 * i;
        case 2: return it.E + 3 * ce + 2 * i;
        case 3: return it.E + 5 * ce + 2 * i;
        case 4: return it.E + 7 * ce + 4 * i;
        case 5: return it.E + 11 * ce + 4 * i;
        default: return it.E + 15 * ce + 2 * i;
    }
}
// states at the start of every interval of channel c from the per-interval (M^len, F): the plain recurrence
// (CPU emulation; k_kw_scan is the warp-parallel form).  stage 0: (M1, F1) -> S1, stage 1: (M2, F2) -> S2.
SS_HD void kw_scan_serial(const LoudItem& it, int c, int stage) {
    double z1 = 0, z2 = 0;
    for (int e = 0; e < it.n_e; ++e) {
        double* s = loud_slot(it, stage ? 6 : 2, c, e);
        s[0] = z1; s[1] = z2;
        const double* m = loud_slot(it, stage ? 5 : 4, c, e);
        const double* f = loud_slot(it, stage ? 3 : 1, c, e);
        const double n1 = m[0] * z1 + m[1] * z2 + f[0], n2 = m[2] * z1 + m[3] * z2 + f[1];
        z1 = n1; z2 = n2;
    }
}
// filter state of one thread = one (channel, interval)
struct KwState { double z1a, z2a, z1b, z2b, acc; };
template <int PASS>
SS_HD void kw_begin(const LoudItem& it, int c, int e, KwState& st) {
    st.z1a = 0; st.z2a = 0; st.z1b = 0; st.z2b = 0; st.acc = 0;
    if (PASS >= 2) { const double* s1 = loud_slot(it, 2, c, e); st.z1a = s1[0]; st.z2a = s1[1]; }
    if (PASS == 3) { const double* s2 = loud_slot(it, 6, c, e); st.z1b = s2[0]; st.z2b = s2[1]; }
}
template <int PASS>
SS_HD void kw_sample(const KCoef& k, float xf, KwState& st) {
    const double x = (double)xf;
    // scipy.signal.lfilter: direct form II transposed, float64; pyloudnorm stores each stage back
    // into the float32 array (meter.py: input_data[:,ch] = filter.apply_filter(...))
    const double y = k.b0[0] * x + st.z1a;
    st.z1a = k.b1[0] * x - k.a1[0] * y + st.z2a;
    st.z2a = k.b2[0] * x - k.a2[0] * y;
    if (PASS >= 2) {
        const double x2 = (double)(float)y;
        const double y2 = k.b0[1] * x2 + st.z1b;
        st.z1b = k.b1[1] * x2 - k.a1[1] * y2 + st.z2b;
        st.z2b = k.b2[1] * x2 - k.a2[1] * y2;
        if (PASS == 3) { const float yf = (float)y2; st.acc += (double)(yf * yf); }
    }
}
template <int PASS>
SS_HD void kw_end(const LoudItem& it, const KCoef& k, int c, int e, const KwState& st) {
    if (PASS == 1) {
        const int len = it.brk[e + 1] - it.brk[e];
        double* f1 = loud_slot(it, 1, c, e); f1[0] = st.z1a; f1[1] = st.z2a;
        const Mat2 m1 = mat_pow(stage_matrix(k, 0), len), m2 = mat_pow(stage_matrix(k, 1), len);
        double* d1 = loud_slot(it, 4, c, e); d1[0] = m1.a; d1[1] = m1.b; d1[2] = m1.c; d1[3] = m1.d;
        double* d2 = loud_slot(it, 5, c, e); d2[0] = m2.a; d2[1] = m2.b; d2[2] = m2.c; d2[3] = m2.d;
    } else if (PASS == 2) {
        double* f2 = loud_slot(it, 3, c, e); f2[0] = st.z1b; f2[1] = st.z2b;
    } else {
        *loud_slot(it, 0, c, e) = st.acc;
    }
}
// one thread, samples read straight from memory (CPU emulation; the CUDA kernel feeds kw_sample from coalesced tiles)
template <int PASS>
SS_HD void kweight_pass(const LoudItem& it, const KCoef& k, int c, int e) {
    const int start = it.brk[e], end = it.brk[e + 1];
    const float* p = it.data + (long long)c * it.stride_c;
    KwState st;
    kw_begin<PASS>(it, c, e, st);
    for (int n = start; n < end; ++n) kw_sample<PASS>(k, p[(long long)n * it.stride_n], st);
    kw_end<PASS>(it, k, c, e, st);
}

// The result of a stem whose target is read on the device (a plan's loudness slot, ss_stream_lufs): the gain of
// loudness_gate for a finite target; NaN for a non-finite one, whose slot is stored unscaled (loud_crop_gain).
SS_HD void loud_result_dev(double lufs, double target, double* result) {
    const double used = isinf(lufs) ? -40.0 : lufs;                                    // SonicSim_audio.py:73-75
    result[0] = lufs;
    result[1] = isfinite(target) ? pow(10.0, (target - used) / 20.0) : NAN;           // pyln.normalize.loudness
}
SS_HD double channel_gain(int c) { return (c == 3 || c == 4) ? 1.41 : 1.0; }   // pyloudnorm G = [1,1,1,1.41,1.41]

// Gating (pyloudnorm meter.py integrated_loudness) for one stem; single thread.
SS_HD void loudness_gate(const LoudItem& it) {
    const int nb = it.n_blocks, C = it.C;
    // pass 1: absolute gate (-70 LUFS) -> per-channel mean of z over the blocks that pass
    double zsum[8]; int cnt = 0;
    for (int c = 0; c < C && c < 8; ++c) zsum[c] = 0;
    for (int pass = 0; pass < 2; ++pass) {
        double gamma_r = -1e300;
        if (pass == 1) {
            double s = 0;
            for (int c = 0; c < C; ++c) s += channel_gain(c) * (cnt ? zsum[c] / cnt : NAN);
            gamma_r = -0.691 + 10.0 * log10(s) - 10.0;        // NaN when no block passes -> nothing passes below
            for (int c = 0; c < C; ++c) zsum[c] = 0;
            cnt = 0;
        }
        for (int j = 0; j < nb; ++j) {
            double zc[8], s = 0;
            for (int c = 0; c < C; ++c) {
                double z = 0;
                for (int e = it.blk_lo[j]; e < it.blk_hi[j]; ++e) z += it.E[(long long)c * it.n_e + e];
                zc[c] = z * it.inv_norm;
                s += channel_gain(c) * zc[c];
            }
            double l = -0.691 + 10.0 * log10(s);
            bool ok = pass == 0 ? (l >= -70.0) : (l > gamma_r && l > -70.0);
            if (ok) { for (int c = 0; c < C; ++c) zsum[c] += zc[c]; ++cnt; }
        }
    }
    double s = 0;
    for (int c = 0; c < C; ++c) s += channel_gain(c) * (cnt ? zsum[c] / cnt : 0.0);   // nan_to_num(mean of empty) = 0
    double lufs = -0.691 + 10.0 * log10(s);                                            // log10(0) = -inf
    if (it.target_dev) { loud_result_dev(lufs, *it.target_dev, it.result); return; }   // (k_loud_gate<true>)
    double used = isinf(lufs) ? -40.0 : lufs;                                          // SonicSim_audio.py:73-75
    it.result[0] = lufs;
    it.result[1] = pow(10.0, (it.target - used) / 20.0);                              // pyln.normalize.loudness
}

}  // namespace ss
