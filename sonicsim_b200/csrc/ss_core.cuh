// sonicsim_b200 :: ss_core.cuh
//
// Per-thread building blocks of the partitioned overlap-save renderer.  Everything here is
// `__host__ __device__` so that tests/emu/ can run the *same* index math and butterflies on
// the CPU, one emulated thread at a time (the authoring container has no GPU).  The CUDA
// kernels in ss_kernels.cu and the emulator in tests/emu/ss_emu.cu share these functions and
// differ only in who loops over `tid` and where the barriers are.
//
// Geometry (fixed): FFT size F = 8192 complex points, partition / block size B = 4096 samples,
// 256 threads per CTA, 32 complex points per thread.  The 8192-point transform is a 3-pass
// Stockham radix-16 x 16 x 16 with the closing radix-2 done in registers (each thread owns
// butterflies j and j+256 of the last pass, whose outputs are exactly a radix-2 pair).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#ifdef __CUDACC__
#define SS_HD __host__ __device__ __forceinline__
#else
#define SS_HD inline
#endif

namespace ss {

constexpr int kF = 8192;          // FFT length (complex points)
constexpr int kB = 4096;          // overlap-save block = RIR partition length (samples / taps)
constexpr int kThreads = 256;     // threads per CTA
constexpr int kSpec = 4096;       // float2 per stored half spectrum; [0] = (DC, Nyquist)
constexpr int kPadF = kF + kF / 16;   // padded smem length in float2

// One float2 of padding per 16: makes the stride-16 scatter of pass A and every other
// half-warp access pattern used below hit 16 distinct 8-byte bank pairs.
SS_HD int pad(int i) { return i + (i >> 4); }

SS_HD float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
// Complex add / subtract, rounded on their own: the compiler must not fuse them with a neighbouring product into an
// FMA, or a source would render to different bits depending on how the butterflies around it were inlined.
#if defined(__CUDA_ARCH__)
SS_HD float2 cadd(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
SS_HD float2 csub(float2 a, float2 b) { return make_float2(__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)); }
#else
SS_HD float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
SS_HD float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
#endif
SS_HD float2 cconj(float2 a) { return make_float2(a.x, -a.y); }
// a + w b, a - w b (4 FMA each) and 2 t - s (2 FMA): a twiddled radix-2 butterfly (t + w b, t - w b) costs
// 6 instructions as (s = cfma(t, w, b), twice_minus(t, s)) instead of 8 as (cmul, cadd, csub).
#if defined(__CUDA_ARCH__)
#define SS_FMA(a, b, c) __fmaf_rn(a, b, c)
#else
#define SS_FMA(a, b, c) ((a) * (b) + (c))
#endif
SS_HD float2 cfma(float2 a, float2 w, float2 b) {
    return make_float2(SS_FMA(-w.y, b.y, SS_FMA(w.x, b.x, a.x)), SS_FMA(w.y, b.x, SS_FMA(w.x, b.y, a.y)));
}
SS_HD float2 cfms(float2 a, float2 w, float2 b) {
    return make_float2(SS_FMA(w.y, b.y, SS_FMA(-w.x, b.x, a.x)), SS_FMA(-w.y, b.x, SS_FMA(-w.x, b.y, a.y)));
}
SS_HD float2 twice_minus(float2 t, float2 s) { return make_float2(SS_FMA(2.f, t.x, -s.x), SS_FMA(2.f, t.y, -s.y)); }
// multiply by -i (forward) or +i (inverse)
template <bool INV> SS_HD float2 rot90(float2 a) { return INV ? make_float2(-a.y, a.x) : make_float2(a.y, -a.x); }
// conjugate the twiddle for the inverse transform
template <bool INV> SS_HD float2 dirw(float2 w) { return INV ? make_float2(w.x, -w.y) : w; }

// Streaming 8-byte load: spectra are read once per CTA, keep them out of L1 so the twiddle tables
// stay resident there.
SS_HD float2 ldg_stream(const float2* p) {
#if defined(__CUDA_ARCH__)
    float2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.f32 {%0, %1}, [%2];" : "=f"(r.x), "=f"(r.y) : "l"(p));
    return r;
#else
    return *p;
#endif
}
SS_HD float2 ldg_cached(const float2* p) {
#if defined(__CUDA_ARCH__)
    return __ldg(p);
#else
    return *p;
#endif
}

// Fire-and-forget accumulate into global memory (second transform of a block that straddles a
// waypoint).  Exactly two addends ever meet at an address and the first was stored by the same
// thread earlier, so the result is order-independent (a + b == b + a in IEEE arithmetic).
SS_HD void red_add(float* p, float v) {
#if defined(__CUDA_ARCH__)
    asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
#else
    *p += v;
#endif
}

// v * g rounded once: the scale k_loud_scale applies to a stored stem (a pooled slot's loudness gain, ss_pool_loudness),
// never contracted into a neighbouring add.  g = 1 returns v's bits.
SS_HD float gain_mul(float v, float g) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(v, g);
#else
    volatile float r = v * g;
    return r;
#endif
}
// The last addend of a sample under a gain g: *p = (*p + v) * g, where *p holds what this thread stored and red_add-ed
// there before.  The sum is rounded as red.global.add.f32 rounds it - to nearest even, subnormal inputs and results
// flushed to sign-preserving zero (add.rn.ftz.f32) - so the result has the bits of red_add(p, v) followed by a scale by
// g.  The load is relaxed at gpu scope, like the RED, so it observes this thread's earlier RED to the same address.
SS_HD void red_add_last(float* p, float v, float g) {
#if defined(__CUDA_ARCH__)
    float a, s;
    asm volatile("ld.relaxed.gpu.global.f32 %0, [%1];" : "=f"(a) : "l"(p) : "memory");
    asm("add.rn.ftz.f32 %0, %1, %2;" : "=f"(s) : "f"(a), "f"(v));
    *p = __fmul_rn(s, g);
#else
    volatile float s = *p + v;
    *p = gain_mul(s, g);
#endif
}

// (1 - w) * a + w * b with every product and the sum rounded separately, like NumPy evaluates
// SonicSim_moving.py:94 (no FMA contraction), so both trajectory forms give identical bits.
SS_HD float lerp_terms(float fa, float a, float fb, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(__fmul_rn(fa, a), __fmul_rn(fb, b));
#else
    volatile float pa = fa * a, pb = fb * b;
    return pa + pb;
#endif
}
// (1 - w) * z.x + w * z.y, the same roundings as lerp_terms(1 - w, z.x, w, z.y)
SS_HD float lerp_pair(float w, float2 z) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(__fmul_rn(__fsub_rn(1.0f, w), z.x), __fmul_rn(w, z.y));
#else
    volatile float omw = 1.0f - w;
    volatile float pa = omw * z.x, pb = w * z.y;
    return pa + pb;
#endif
}
SS_HD float one_minus(float w) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(1.0f, w);
#else
    return 1.0f - w;
#endif
}

// Twiddle tables (forward sign, filled in double precision on the host):
//   tw [m]           = exp(-2 pi i m / 8192)            m < 8192   (closing radix-2)
//   twB[r * 16 + k]  = exp(-2 pi i k r / 256)           r, k < 16  (pass B)
//   twC[r * 256 + k] = exp(-2 pi i k r / 4096)          r < 16, k < 256 (pass C)
// r-major so that a warp (consecutive k) reads consecutive words.
struct Tables { const float2* tw; const float2* twB; const float2* twC; };
#ifndef SS_TWC_STREAM_FROM
#define SS_TWC_STREAM_FROM 16      // rows >= this of the pass-C table bypass L1 (experiment knob)
#endif
constexpr int kTabB = 16 * 16, kTabC = 16 * 256;

template <bool INV>
SS_HD void fft4(float2& v0, float2& v1, float2& v2, float2& v3) {
    float2 a0 = cadd(v0, v2), a1 = csub(v0, v2), a2 = cadd(v1, v3), a3 = rot90<INV>(csub(v1, v3));
    v0 = cadd(a0, a2); v2 = csub(a0, a2); v1 = cadd(a1, a3); v3 = csub(a1, a3);
}

// radix-4 butterfly whose inputs 1..3 still have to be multiplied by w1..w3 (input 0 by w0 when TW0):
// the products are folded into the first add/sub level.
template <bool INV, bool TW0>
SS_HD void fft4_tw(float2& v0, float2& v1, float2& v2, float2& v3, float2 w0, float2 w1, float2 w2, float2 w3) {
    const float2 t0 = TW0 ? cmul(v0, w0) : v0;
    const float2 a0 = cfma(t0, w2, v2), a1 = twice_minus(t0, a0);
    const float2 t1 = cmul(v1, w1);
    const float2 a2 = cfma(t1, w3, v3), a3 = rot90<INV>(twice_minus(t1, a2));
    v0 = cadd(a0, a2); v2 = csub(a0, a2); v1 = cadd(a1, a3); v3 = csub(a1, a3);
}

// second level of fft16: v[4a + c] *= W16^(a c) folded into the radix-4 butterflies (forward W16 = exp(-2 pi i / 16))
template <bool INV>
SS_HD void fft16_level2(float2 (&v)[16]) {
    const float C1 = 0.92387953251128674f, S1 = 0.38268343236508977f, H = 0.70710678118654752f;
    const float2 one = make_float2(1.f, 0.f);
    fft4<INV>(v[0], v[1], v[2], v[3]);
    fft4_tw<INV, false>(v[4], v[5], v[6], v[7], one, dirw<INV>(make_float2(C1, -S1)), dirw<INV>(make_float2(H, -H)),
                        dirw<INV>(make_float2(S1, -C1)));                                   // a = 1: W^1, W^2, W^3
    {                                                                                       // a = 2: W^2, W^4 = -+i, W^6
        const float2 r2 = rot90<INV>(v[10]);
        const float2 a0 = cadd(v[8], r2), a1 = csub(v[8], r2);
        const float2 t1 = cmul(v[9], dirw<INV>(make_float2(H, -H)));
        const float2 a2 = cfma(t1, dirw<INV>(make_float2(-H, -H)), v[11]), a3 = rot90<INV>(twice_minus(t1, a2));
        v[8] = cadd(a0, a2); v[10] = csub(a0, a2); v[9] = cadd(a1, a3); v[11] = csub(a1, a3);
    }
    fft4_tw<INV, false>(v[12], v[13], v[14], v[15], one, dirw<INV>(make_float2(S1, -C1)), dirw<INV>(make_float2(-H, -H)),
                        dirw<INV>(make_float2(-C1, S1)));                                   // a = 3: W^3, W^6, W^9
}

// In-register 16-point DFT (4 x 4).  Input natural order v[n]; output X[a + 4c] is left in
// v[4a + c] (see out16()).
template <bool INV>
SS_HD void fft16(float2 (&v)[16]) {
#pragma unroll
    for (int b = 0; b < 4; ++b) fft4<INV>(v[b], v[b + 4], v[b + 8], v[b + 12]);
    fft16_level2<INV>(v);
}
// the same with the inter-pass twiddles v[r] *= w[r], r = 1..15, folded into the first level.  The twiddles of a
// thread's two butterflies of a pass (j and j + 256) are the same, and they do not depend on the data: tw_load can be
// issued ahead of the barrier that guards the pass's inputs.
template <bool INV, int STRIDE>
SS_HD void tw_load(const float2* tab, float2 (&w)[16]) {
    w[0] = make_float2(1.f, 0.f);
#pragma unroll
    for (int r = 1; r < 16; ++r)
        w[r] = dirw<INV>((STRIDE == 256 && r >= SS_TWC_STREAM_FROM) ? ldg_stream(tab + r * STRIDE) : ldg_cached(tab + r * STRIDE));
}
// only rows 1, 2, 4, 8 of the table are loaded, the other eleven twiddles are products of them
// (w_3 = w_1 w_2, ..., w_(8 + r) = w_r w_8): 11 complex multiplies instead of 11 loads through the L1 data pipe
template <bool INV, int STRIDE>
SS_HD void tw_load_pow(const float2* tab, float2 (&w)[16]) {
    w[0] = make_float2(1.f, 0.f);
    w[1] = dirw<INV>(ldg_cached(tab + 1 * STRIDE));
    w[2] = dirw<INV>(ldg_cached(tab + 2 * STRIDE));
    w[4] = dirw<INV>(ldg_cached(tab + 4 * STRIDE));
    w[8] = dirw<INV>(ldg_cached(tab + 8 * STRIDE));
    w[3] = cmul(w[1], w[2]); w[5] = cmul(w[1], w[4]); w[6] = cmul(w[2], w[4]); w[7] = cmul(w[3], w[4]);
#pragma unroll
    for (int r = 1; r < 8; ++r) w[8 + r] = cmul(w[r], w[8]);
}
template <bool INV>
SS_HD void fft16_w(float2 (&v)[16], const float2 (&w)[16]) {
    fft4_tw<INV, false>(v[0], v[4], v[8], v[12], w[0], w[4], w[8], w[12]);
#pragma unroll
    for (int b = 1; b < 4; ++b) fft4_tw<INV, true>(v[b], v[b + 4], v[b + 8], v[b + 12], w[b], w[b + 4], w[b + 8], w[b + 12]);
    fft16_level2<INV>(v);
}
// Every transform of the library (forward and inverse, every kernel variant, and the CPU emulation) gets its
// inter-pass twiddles the same way, so that a source renders to the same bits whatever batch it is part of.
#ifndef SS_TWPOW
#define SS_TWPOW 1            // 1: rows 1, 2, 4, 8 of the table + 11 products (fewer bytes through the L1 data pipe, the
                              //    scarcer resource); 0: all fifteen loaded from the table
#endif
template <bool INV, int STRIDE>
SS_HD void tw_get(const float2* tab, float2 (&w)[16]) {
#if SS_TWPOW
    tw_load_pow<INV, STRIDE>(tab, w);
#else
    tw_load<INV, STRIDE>(tab, w);
#endif
}
template <bool INV, int STRIDE>
SS_HD void fft16_tw(float2 (&v)[16], const float2* tab) {
    float2 w[16];
    tw_get<INV, STRIDE>(tab, w);
    fft16_w<INV>(v, w);
}
// register slot that holds output index r after fft16
SS_HD constexpr int out16(int r) { return 4 * (r & 3) + (r >> 2); }

// ---------------------------------------------------------------------------------------
// Stockham passes on a padded shared-memory array `s` (float2[kPadF]).
// `tw` is the table exp(-2 pi i m / 8192), m in [0, 8192).
// Butterfly j of a pass with sub-length Ns reads s[j + 512 r] and writes
// s[(j / Ns) * 16 Ns + (j % Ns) + r Ns].
// ---------------------------------------------------------------------------------------

// Pass A (Ns = 1) store: v holds fft16 outputs of butterfly j (no input twiddles when Ns = 1).
// pad(16 j + r) = 17 j + r.
SS_HD void passA_store(float2* s, int j, const float2 (&v)[16]) {
    float2* d = s + 17 * j;
#pragma unroll
    for (int r = 0; r < 16; ++r) d[r] = v[out16(r)];
}

// pad(j + 512 r) = pad(j) + 544 r
SS_HD void pass_load(const float2* s, int j, float2 (&v)[16]) {
    const float2* p = s + pad(j);
#pragma unroll
    for (int r = 0; r < 16; ++r) v[r] = p[544 * r];
}

// Pass B (Ns = 16): twiddle exp(-+2 pi i k r / 256), k = j % 16
template <bool INV>
SS_HD void passB_compute(int j, float2 (&v)[16], const Tables& T) {
    fft16_tw<INV, 16>(v, T.twB + (j & 15));
}
// destination (j / 16) * 256 + (j % 16) + 16 r, padded = (j / 16) * 272 + (j % 16) + 17 r
SS_HD void passB_store(float2* s, int j, const float2 (&v)[16]) {
    float2* d = s + (j >> 4) * 272 + (j & 15);
#pragma unroll
    for (int r = 0; r < 16; ++r) d[17 * r] = v[out16(r)];
}

// Pass C (Ns = 256): twiddle exp(-+2 pi i k r / 4096), k = j % 256.  Outputs stay in registers:
// butterfly j (< 256) yields natural-order points j + 256 r of the first half-length transform,
// butterfly j + 256 the same points of the second one.
template <bool INV>
SS_HD void passC_compute(int j, float2 (&v)[16], const Tables& T) {
    fft16_tw<INV, 256>(v, T.twC + (j & 255));
}

// Closing radix-2 (Ns = 4096) for thread t: lo/hi are the pass-C results of butterflies t and t+256.
// Returns through lo[slot] the points t + 256 r and through hi[slot] the points 4096 + t + 256 r,
// slot = out16(r).
// u[r] = exp(-+2 pi i (t + 256 r) / 8192) = wt * exp(-+2 pi i r / 32), r < 16 (wt = tw[t], already
// direction-adjusted): seven products, the upper eight are quarter-turn rotations of the lower eight.
template <bool INV>
SS_HD void final_twiddles(float2 wt, float2 (&u)[16]) {
    const float c32[8] = {1.f, 0.98078528040323043f, 0.92387953251128674f, 0.83146961230254524f,
                          0.70710678118654752f, 0.55557023301960218f, 0.38268343236508977f, 0.19509032201612825f};
    const float s32[8] = {0.f, 0.19509032201612825f, 0.38268343236508977f, 0.55557023301960218f,
                          0.70710678118654752f, 0.83146961230254524f, 0.92387953251128674f, 0.98078528040323043f};
    u[0] = wt;
#pragma unroll
    for (int r = 1; r < 8; ++r) u[r] = cmul(wt, make_float2(c32[r], INV ? s32[r] : -s32[r]));
#pragma unroll
    for (int r = 0; r < 8; ++r) u[r + 8] = rot90<INV>(u[r]);
}

// ---------------------------------------------------------------------------------------
// Spectrum-domain helpers.
//   stored half spectrum S[0] = (DC, Nyquist), S[k] = bin k for 1 <= k < 4096.
// For a pair of real sequences (a, b) convolved with real x:  z = x*a + i x*b,
//   Z[k]   = P + iQ,  Z[F-k] = conj(P) + i conj(Q),   P = X[k] A[k], Q = X[k] B[k].
// ---------------------------------------------------------------------------------------
SS_HD float2 z_direct(float2 P, float2 Q) { return make_float2(P.x - Q.y, P.y + Q.x); }
SS_HD float2 z_mirror(float2 P, float2 Q) { return make_float2(P.x + Q.y, Q.x - P.y); }
SS_HD void cmac(float2& acc, float2 a, float2 b) {
    acc.x += a.x * b.x - a.y * b.y;
    acc.y += a.x * b.y + a.y * b.x;
}

// Ownership of pass-A butterflies: thread t (1..255) owns jA = t and jB = 512 - t; thread 0 owns
// jA = 0 and jB = 256.  With that choice every bin k < 4096 a thread loads also supplies the
// mirrored bin F - k of one of its own butterflies, so each spectrum word is read exactly once.
SS_HD int passA_jA(int t) { return t; }
SS_HD int passA_jB(int t) { return t == 0 ? 256 : 512 - t; }

// ---------------------------------------------------------------------------------------
// Trajectory helpers (compact form of SonicSim_moving.setup_dynamic_interp's (idx, w)):
//   bounds[0..S], bounds[0] = 0, bounds[S] = N, segment s covers [bounds[s], bounds[s+1]).
// ---------------------------------------------------------------------------------------
SS_HD int seg_of(const int* bounds, int S, int n) {
    // number of i in [1, S] with bounds[i] <= n  (skips empty segments like np.repeat does)
    int lo = 0, hi = S;            // answer in [lo, hi]
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (bounds[mid] <= n) lo = mid; else hi = mid - 1;
    }
    return lo < S ? lo : S - 1;    // n == N cannot happen for valid samples; clamp anyway
}
// np.linspace(0, 1, num, endpoint=False)[i].astype(float32): float64 i * (1/num), then rounded.
SS_HD float seg_weight(int i, int num) {
    double step = 1.0 / (double)num;
    return (float)((double)i * step);
}

}  // namespace ss
