// tests/emu/ss_emu_taps.cu - tap-form host banks (SS_BANK_TAPS) in the emulated kernels: the stored rows and their
// transform.
//
// TEST INFRASTRUCTURE, like ss_emu_stage.cu, whose bank builder, stage_set and stage_cap it reuses (included below).
// A tap bank is built as the library builds it: k_rir_absmax / k_rir_direct over bank_build's blockless source, then
// tap_value for every stored tap.  A staged row range is transformed as the plan's transform launch does it: k_prepare's
// CTAs over tap_source, with the plan-time CTA count.  Built with g++ (`-x c++`) by tests/test_taps_pool.py.
#include "ss_emu_stage.cu"

extern "C" {

// The rows of a tap bank of one RIR set (P, C, L): rows receives P*C*K * 4096 float32, cut the P*C direct-path row
// lengths (direct_taps > 0).
int emu_tap_bank(const float* rir, int P, int C, int L, int normalize, int direct_taps, float* rows, int* cut) {
    Source S;
    memset(&S, 0, sizeof(S));
    S.rir = rir; S.N = 1; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = 1;
    S.mode = P == 1 ? MODE_STATIC : MODE_MOVING_BOUNDS;
    std::vector<float> norm_part(kNormParts);
    if (normalize) S.norm_part = norm_part.data();
    if (direct_taps > 0) { S.cut = cut; S.direct_taps = direct_taps; }
    emu_rir_prep(S, norm_part.data());
    const float m = S.norm_part ? rir_absmax(S) : 0.f;
    for (int row = 0; row < P * C * S.K; ++row)
        for (int j = 0; j < kB; ++j) rows[(size_t)row * kB + j] = tap_value(S, row, j, m);
    return 0;
}

// The transform of one staged row range: `staged` holds the candidate's P*C*K rows of taps where only rows
// [row0, row0 + rows) are the bank's (the caller puts NaN in every other row, so that a read outside shows), spec the
// staging area's sets * rows_cap spectra rows.  Runs k_prepare's CTAs 0 .. sets * ceil(rows_cap / 2) - 1 over
// tap_source (cut: the bank's cut table for sets == 2).  info receives [spectra_pairs_h, CTAs that transformed a row
// pair, CTAs that took the block branch and returned at counts[0] == 0, rows_stored_h, h_row0].
int emu_tap_transform(const float* staged, const int* cut, int P, int C, int K, int row0, int rows, int sets,
                      int rows_cap, float2* spec, int* info) {
    const Tables& T = tables();
    int zero = 0;
    const Source S = tap_source(staged + (size_t)row0 * kB, spec, sets > 1 ? const_cast<int*>(cut) : nullptr, P, C, K,
                                row0, rows, &zero);
    const int nh = spectra_pairs_h(S), nx = spectra_pairs_x(S), ctas = sets * ((rows_cap + 1) >> 1);
    int transformed = 0, returned = 0;
    for (int local = 0; local < ctas; ++local) {
        if (local >= nh + nx) {
            // k_prepare's block branch, restated: its first read is counts[0] (`if (blk >= S.counts[0]) return;`), before
            // the block table or anything else, so a CTA here returns at once when every warp's blk >= counts[0]
            bool all = true;
            for (int warp = 0; warp < kThreads / 32; ++warp) all = all && (local - nh - nx) * 8 + warp >= S.counts[0];
            returned += all ? 1 : 0;
            continue;
        }
        cta_spectra(S, local, T);
        ++transformed;
    }
    info[0] = nh; info[1] = transformed; info[2] = returned; info[3] = rows_stored_h(S); info[4] = S.h_row0;
    return 0;
}

// stage_area(sets, rows_cap, nx, taps): out = [view, spec, x, taps, end]
int emu_stage_area(int sets, int rows_cap, int nx, int taps, int64_t* out) {
    const StageArea a = stage_area(sets, rows_cap, nx, taps != 0);
    out[0] = (int64_t)a.view; out[1] = (int64_t)a.spec; out[2] = (int64_t)a.x; out[3] = (int64_t)a.taps;
    out[4] = (int64_t)a.end;
    return 0;
}

// tap_block(at, n_staged, n_tap): out = [taps, src, prefix, zero, end]; sizes = [sizeof StageTap, sizeof Source]
int emu_tap_block(int64_t at, int n_staged, int n_tap, int64_t* out, int64_t* sizes) {
    const TapBlock t = tap_block((size_t)at, n_staged, n_tap);
    out[0] = (int64_t)t.taps; out[1] = (int64_t)t.src; out[2] = (int64_t)t.prefix; out[3] = (int64_t)t.zero;
    out[4] = (int64_t)t.end;
    sizes[0] = (int64_t)sizeof(StageTap); sizes[1] = (int64_t)sizeof(Source);
    return 0;
}

}  // extern "C"
