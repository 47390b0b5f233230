// tests/emu/ss_emu_bank.cu - CPU emulation of RIR spectrum banks (ss_bank): building one, rendering from it.
//
// TEST INFRASTRUCTURE, like the other emulations, whose phases it reuses (included below).  A bank is built as the
// library builds it: k_rir_absmax / k_rir_direct / k_prepare's RIR CTAs over a source without blocks (nblk_max = 0).  A
// banked source (set_banked: no rir, spectra and cuts from the bank) then runs k_prepare's dry-window CTAs and range warps
// (fill_items) and the render CTAs, whole or windowed.  Built with g++ (`-x c++`) by tests/test_bank.py; the library also
// exports emu_render, emu_render_dual and emu_render_window, the references of that test.
#include "ss_emu_window.cu"

extern "C" {

// The bank of one RIR set (P, C, L): spec receives (direct_taps > 0 ? 2 : 1) * P*C*K * 4096 complex64, cut the P*C
// direct-path row lengths (direct_taps > 0).  Returns the number of k_prepare CTAs run.
int emu_bank_create(const float* rir, int P, int C, int L, int normalize, int direct_taps, float2* spec, int* cut) {
    const Tables& T = tables();
    Source S;
    memset(&S, 0, sizeof(S));
    S.rir = rir; S.N = 1; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = 1;
    S.mode = P == 1 ? MODE_STATIC : MODE_MOVING_BOUNDS;
    S.nblk_max = 0;
    S.hspec = spec;
    std::vector<float> norm_part(kNormParts);
    if (normalize) S.norm_part = norm_part.data();
    if (direct_taps > 0) { S.cut = cut; S.direct_taps = direct_taps; }
    emu_rir_prep(S, norm_part.data());
    const int ns = spectra_pairs_h(S) + spectra_pairs_x(S) + range_ctas(S);
    for (int i = 0; i < ns; ++i) cta_spectra(S, i, T);
    return ns;
}

// A banked source rendered into out (C, N) - or (C, win_len) with win_len > 0 - [and out_direct when direct_taps > 0,
// which must then be the bank's].  No RIR pointer exists here.  stats (may be null) receives [RIR pair CTAs of k_prepare,
// dry-window pair CTAs, render items].
int emu_render_banked(const float* x, const float2* spec, const int* cut, float* out, const int32_t* bounds,
                      const int32_t* idx, const float* w, int N, int P, int C, int L, int mode, int aligned,
                      int win_start, int win_len, float* out_direct, int direct_taps, int* stats) {
    emu_source(x, nullptr, spec, cut, out, bounds, idx, w, N, P, C, L, mode, aligned, win_start, win_len, out_direct,
               direct_taps, 0, 0, nullptr, stats);
    return 0;
}

}  // extern "C"
