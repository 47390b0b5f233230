// tests/emu/ss_emu_window.cu - CPU emulation of a windowed source (ss_source.win_start / win_len).
//
// TEST INFRASTRUCTURE, like ss_emu.cu and ss_emu_dual.cu, whose emulated phases it reuses (included below): the full
// plan's blocks cut to the window by the kernels' window_blocks / window_span, the RIR rows of window_rows, k_prepare's
// spectra CTAs (rows_of_pair_h, make_row_x over the windowed table) and range warps (the kept-block test, fill_items
// with its clipped store range and window-relative rows), and the render CTAs with their epilogues.  Built with g++
// (`-x c++`) by tests/test_window.py.
#include "ss_emu_dual.cu"

// The full plan's blocks in use, ascending (k_blocks / the host's full_blocks)
static int emu_full_blocks(const Source& S, Block* blocks) {
    int nblk = 0;
    if (S.aligned) {
        for (int sg = 0; sg < S.P - 1; ++sg) {
            const int b0 = S.bounds[sg], n_s = S.bounds[sg + 1] - b0;
            for (int q = 0; q < seg_blocks(n_s); ++q) {
                Block bk; bk.start = b0 + kB * q; bk.len = n_s - kB * q < kB ? n_s - kB * q : kB; bk.p_lo = sg; bk.p_hi = sg + 1;
                blocks[nblk++] = bk;
            }
        }
    } else {
        nblk = S.nb;
        for (int bi = 0; bi < nblk; ++bi) {
            Block bk; bk.start = bi * kB; bk.len = S.N - bi * kB < kB ? S.N - bi * kB : kB; bk.p_lo = 0; bk.p_hi = 0;
            blocks[bi] = bk;
        }
    }
    return nblk;
}

// k_prepare's range warps for a windowed source: blocks outside the window get no items
static void prepare_ranges_window(const Source& S, RItem* items) {
    for (int blk = 0; blk < S.counts[0]; ++blk) {
        if ((unsigned)(blk - win_first(S)) >= (unsigned)win_blocks(S)) continue;
        Block bk = S.blocks[blk];
        if (S.mode == MODE_MOVING_BOUNDS && !S.aligned) {
            bk.p_lo = seg_of(S.bounds, S.P - 1, bk.start);
            bk.p_hi = seg_of(S.bounds, S.P - 1, bk.start + bk.len - 1) + 1;
        } else if (S.mode == MODE_MOVING_INDEXED) {
            int pmin = 0x7fffffff, pmax = -1;
            for (int n = bk.start; n < bk.start + bk.len; ++n) { int v = S.idx[n]; pmin = v < pmin ? v : pmin; pmax = v > pmax ? v : pmax; }
            bk.p_lo = pmin < 0 ? 0 : pmin;
            bk.p_hi = pmax + 1 > S.P - 1 ? S.P - 1 : pmax + 1;
        }
        for (int lane = 0; lane < 32; ++lane) fill_items(S, items, blk, bk, lane, 32);
    }
}

extern "C" {

// Windowed render of one source into out (C, win_len) [and out_direct (C, win_len) when direct_taps > 0].
// aligned: the blocking plan (the library chooses it over the whole trajectory, ss_debug_plan reports it);
// restrict_rows: transform only the RIR rows of the positions the window's blocks touch (the library does so when the
// trajectory is visible on the host), else all of them.  stats (may be null) receives
// [table blocks, kept blocks, first RIR row, RIR rows per set].
int emu_render_window(const float* x, const float* rir, float* out, const int32_t* bounds, const int32_t* idx,
                      const float* w, int N, int P, int C, int L, int mode, int aligned, int win_start, int win_len,
                      float* out_direct, int direct_taps, int normalize, int restrict_rows, int* stats) {
    const Tables& T = tables();
    Source S;
    memset(&S, 0, sizeof(S));
    S.x = x; S.rir = rir; S.out = out; S.bounds = bounds; S.idx = idx; S.w = w;
    S.N = N; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = (N + kB - 1) / kB; S.mode = mode;
    S.aligned = aligned;
    std::vector<Block> full(S.aligned ? S.nb + P - 1 : S.nb);
    const int nfull = emu_full_blocks(S, full.data());
    const WinSpan ws = window_blocks(full.data(), nfull, win_start, win_start + win_len, S.K);
    S.nblk_max = ws.g1 - ws.g0;
    // RIR positions the kept blocks interpolate between
    int pa = 0, pb = P - 1;
    if (mode == MODE_STATIC) pb = 0;
    else if (restrict_rows && mode == MODE_MOVING_BOUNDS) {
        const Block &b0 = full[ws.k0], &b1 = full[ws.k1 - 1];
        if (S.aligned) { pa = b0.p_lo; pb = b1.p_hi; }
        else { pa = seg_of(bounds, P - 1, b0.start); pb = seg_of(bounds, P - 1, b1.start + b1.len - 1) + 1; }
    }
    window_rows(P, C, S.K, pa, pb, S.h_row0, S.h_rows);
    const int sets = direct_taps > 0 ? 2 : 1;
    std::vector<float2> hs((size_t)sets * S.h_rows * kSpec), xs((size_t)S.nblk_max * kSpec);
    std::vector<Block> blocks(S.nblk_max);
    for (int i = 0; i < S.nblk_max; ++i) blocks[i] = full[ws.g0 + i];
    std::vector<double> rstep(P);
    if (mode == MODE_MOVING_BOUNDS)
        for (int sg = 0; sg < P - 1; ++sg) rstep[sg] = 1.0 / (double)(bounds[sg + 1] - bounds[sg]);
    std::vector<float> norm_part(kNormParts);
    std::vector<int> cut((size_t)P * C);
    int counts[8] = {S.nblk_max, 0, ws.k0 - ws.g0, ws.k1 - ws.k0, win_start, win_len, 0, 0};
    S.hspec = hs.data(); S.xspec = xs.data(); S.blocks = blocks.data(); S.rstep = rstep.data(); S.counts = counts;
    if (normalize) S.norm_part = norm_part.data();
    if (direct_taps > 0) { S.cut = cut.data(); S.out_direct = out_direct; S.direct_taps = direct_taps; }
    std::vector<RItem> items((size_t)S.nblk_max * items_per_block(S));
    emu_rir_prep(S, norm_part.data());
    const int ns = spectra_pairs_h(S) + spectra_pairs_x(S);
    for (int i = 0; i < ns; ++i) cta_spectra_sets(S, i, T);
    prepare_ranges_window(S, items.data());
    const int nr = win_blocks(S) * items_per_block(S);
    const int grid = nr < 3 ? nr : 3;
    for (int cta = 0; cta < grid; ++cta) {
        if (S.aligned || (mode == MODE_STATIC && S.K == 1)) cta_render_fast(items.data(), nr, cta, grid, T);
        else cta_render(items.data(), nr, cta, grid, T, false, S.K > 1);
    }
    if (stats) { stats[0] = S.nblk_max; stats[1] = ws.k1 - ws.k0; stats[2] = S.h_row0; stats[3] = S.h_rows; }
    return 0;
}

}  // extern "C"
