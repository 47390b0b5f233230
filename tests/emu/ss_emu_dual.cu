// tests/emu/ss_emu_dual.cu - CPU emulation of a source with SS_DIRECT_TARGET (and optionally SS_RIR_NORMALIZE).
//
// TEST INFRASTRUCTURE, like ss_emu.cu, whose emulated phases it reuses (included below): k_rir_absmax / k_rir_direct
// (the shared per-row scan peak_scan), k_prepare's RIR rows of both sets (rows_of_pair_h), its range warps (fill_items,
// which emits the direct items) and the render CTAs.  Built with g++ (`-x c++`) by tests/test_direct_target.py.
#include "ss_emu.cu"

// k_rir_absmax (all partial maxima in slot 0) and k_rir_direct, one emulated lane per row
static void emu_rir_prep(const Source& S, float* norm_part) {
    if (S.norm_part) {
        float m = 0.f;
        for (size_t i = 0; i < (size_t)S.P * S.C * S.L; ++i) m = fabsf(S.rir[i]) > m ? fabsf(S.rir[i]) : m;
        for (int i = 0; i < kNormParts; ++i) norm_part[i] = i == 0 ? m : 0.f;
    }
    if (S.cut) {
        const float div = S.norm_part ? rir_absmax(S) : 0.f;
        for (int row = 0; row < S.P * S.C; ++row)
            S.cut[row] = direct_cut(peak_scan(S.rir + (size_t)row * S.L, S.L, div, 0, 1).i, S.L, S.direct_taps);
    }
}

// one k_prepare spectra CTA, rows chosen as the kernel chooses them (reverberant pairs, then direct pairs)
static void cta_spectra_sets(const Source& S, int local, const Tables& T) {
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

extern "C" {

// emu_render's launches for one source with SS_DIRECT_TARGET (direct-path stem into out_direct, direct_taps >= 1)
// and, if `normalize`, SS_RIR_NORMALIZE: [k_rir_absmax,] k_rir_direct, k_prepare, k_render.
int emu_render_dual(const float* x, const float* rir, float* out, const int32_t* bounds, const int32_t* idx,
                    const float* w, int N, int P, int C, int L, int mode, float* out_direct, int direct_taps,
                    int normalize) {
    const Tables& T = tables();
    Source S;
    memset(&S, 0, sizeof(S));
    S.x = x; S.rir = rir; S.out = out; S.bounds = bounds; S.idx = idx; S.w = w;
    S.N = N; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = (N + kB - 1) / kB; S.mode = mode;
    S.aligned = (mode == MODE_MOVING_BOUNDS && S.K == 1) ? 1 : 0;
    S.nblk_max = S.aligned ? S.nb + P - 1 : S.nb;
    std::vector<float2> hs((size_t)2 * P * C * S.K * kSpec), xs((size_t)S.nblk_max * kSpec);
    std::vector<Block> blocks(S.nblk_max);
    std::vector<double> rstep(P);
    std::vector<float> norm_part(kNormParts);
    std::vector<int> cut((size_t)P * C);
    int counts[2] = {0, 0};
    S.hspec = hs.data(); S.xspec = xs.data(); S.blocks = blocks.data(); S.rstep = rstep.data(); S.counts = counts;
    if (normalize) S.norm_part = norm_part.data();
    S.cut = cut.data(); S.out_direct = out_direct; S.direct_taps = direct_taps;
    std::vector<RItem> items(max_render_items(S));
    emu_rir_prep(S, norm_part.data());
    emu_blocks(S);
    const int ns = spectra_pairs_h(S) + spectra_pairs_x(S);
    for (int i = 0; i < ns; ++i) cta_spectra_sets(S, i, T);
    prepare_ranges(S, items.data());
    const int nr = counts[0] * items_per_block(S);
    const int grid = nr < 3 ? nr : 3;              // a few persistent CTAs, each looping over many items
    for (int cta = 0; cta < grid; ++cta) {
        if (S.aligned || (mode == MODE_STATIC && S.K == 1)) cta_render_fast(items.data(), nr, cta, grid, T);
        else cta_render(items.data(), nr, cta, grid, T, false, S.K > 1);
    }
    return 0;
}

}  // extern "C"
