// tests/emu/ss_emu_window.cu - CPU emulation of a windowed source (ss_source.win_start / win_len).
//
// TEST INFRASTRUCTURE, like ss_emu.cu and ss_emu_dual.cu, whose emulated source driver it runs (included below): the
// full plan's blocks cut to the window by the kernels' window_blocks / window_span, the RIR rows of window_rows,
// k_prepare's spectra CTAs (rows_of_pair_h, make_row_x over the windowed table) and range warps (the kept-block test,
// fill_items with its clipped store range and window-relative rows), and the render CTAs with their epilogues.  Built
// with g++ (`-x c++`) by tests/test_window.py.
#include "ss_emu_dual.cu"

extern "C" {

// Windowed render of one source into out (C, win_len) [and out_direct (C, win_len) when direct_taps > 0].
// aligned: the blocking plan (the library chooses it over the whole trajectory, ss_debug_plan reports it);
// restrict_rows: transform only the RIR rows of the positions the window's blocks touch (the library does so when the
// trajectory is visible on the host), else all of them.  stats (may be null) receives
// [table blocks, kept blocks, first RIR row, RIR rows per set].
int emu_render_window(const float* x, const float* rir, float* out, const int32_t* bounds, const int32_t* idx,
                      const float* w, int N, int P, int C, int L, int mode, int aligned, int win_start, int win_len,
                      float* out_direct, int direct_taps, int normalize, int restrict_rows, int* stats) {
    emu_source(x, rir, nullptr, nullptr, out, bounds, idx, w, N, P, C, L, mode, aligned, win_start, win_len, out_direct,
               direct_taps, normalize, restrict_rows, stats, nullptr);
    return 0;
}

}  // extern "C"
