// tests/emu/ss_emu_dual.cu - CPU emulation of a source with SS_DIRECT_TARGET (and optionally SS_RIR_NORMALIZE).
//
// TEST INFRASTRUCTURE, like ss_emu.cu, whose emulated source driver it runs (included below): k_rir_absmax /
// k_rir_direct (the shared per-row scan peak_scan), k_prepare's RIR rows of both sets (rows_of_pair_h), its range warps
// (fill_items, which emits the direct items) and the render CTAs.  Built with g++ (`-x c++`) by
// tests/test_direct_target.py.
#include "ss_emu.cu"

extern "C" {

// emu_render's launches for one source with SS_DIRECT_TARGET (direct-path stem into out_direct, direct_taps >= 1)
// and, if `normalize`, SS_RIR_NORMALIZE: [k_rir_absmax,] k_rir_direct, k_prepare, k_render.
int emu_render_dual(const float* x, const float* rir, float* out, const int32_t* bounds, const int32_t* idx,
                    const float* w, int N, int P, int C, int L, int mode, float* out_direct, int direct_taps,
                    int normalize) {
    const int aligned = mode == MODE_MOVING_BOUNDS && (L + kB - 1) / kB == 1;
    emu_source(x, rir, nullptr, nullptr, out, bounds, idx, w, N, P, C, L, mode, aligned, 0, 0, out_direct, direct_taps,
               normalize, 0, nullptr, nullptr);
    return 0;
}

}  // extern "C"
