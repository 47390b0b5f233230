// tests/emu/ss_emu_stream_loud.cu - the loudness slots of plans (ss_stream_lufs) in the emulated kernels: the gate of
// k_loud_gate<true>, which reads its target from memory (loud_result_dev), and k_loud_crop's per-thread code
// (loud_crop_head, loud_crop_sample).
//
// TEST INFRASTRUCTURE, like ss_emu.cu.  Built with g++ (`-x c++`) by tests/test_stream_loudness.py.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"
#include "../../sonicsim_b200/csrc/ss_loud.cuh"

using namespace ss;

extern "C" {

// k_kweight<1..3>, the scans and k_loud_gate<true> over a (C, N) stem whose target is read from *target: result
// receives (LUFS, gain)
int emu_lufs_dev(const float* data, int N, int C, double rate, double block_size, const double* target,
                 const int32_t* brk, int n_e, const int32_t* blk_lo, const int32_t* blk_hi, int n_blocks,
                 double* result) {
    LoudItem it; memset(&it, 0, sizeof(it));
    std::vector<double> E((size_t)kLoudScratch * C * n_e);
    it.data = data; it.brk = brk; it.blk_lo = blk_lo; it.blk_hi = blk_hi; it.E = E.data(); it.result = result;
    it.stride_n = 1; it.stride_c = N; it.N = N; it.C = C; it.n_e = n_e; it.n_blocks = n_blocks;
    it.inv_norm = 1.0 / (block_size * rate); it.target_dev = target;
    const KCoef k = make_kcoef(rate);
    for (int c = 0; c < C; ++c) for (int e = 0; e < n_e; ++e) kweight_pass<1>(it, k, c, e);
    for (int c = 0; c < C; ++c) kw_scan_serial(it, c, 0);
    for (int c = 0; c < C; ++c) for (int e = 0; e < n_e; ++e) kweight_pass<2>(it, k, c, e);
    for (int c = 0; c < C; ++c) kw_scan_serial(it, c, 1);
    for (int c = 0; c < C; ++c) for (int e = 0; e < n_e; ++e) kweight_pass<3>(it, k, c, e);
    loudness_gate(it);
    return 0;
}

// k_loud_crop of one slot: the crops of the (C, N) whole stems into out / out_dir (C, len; out_dir may be null);
// returns the error bits the kernel reports and *start_out the start it cut at
int emu_loud_crop(const float* whole, const float* whole_dir, float* out, float* out_dir, const int* ws_dev, int ws,
                  int len, int N, int C, const double* target, const double* result, int* start_out) {
    const LoudCrop q = {whole, whole_dir, out, out_dir, ws_dev, target, result, ws, len, N, C};
    int start;
    float g;
    const unsigned err = loud_crop_head(q, start, g);
    for (int dir = 0; dir < 2; ++dir) {
        float* const dst = dir ? out_dir : out;
        if (dst) for (long long i = 0; i < (long long)C * len; ++i) dst[i] = loud_crop_sample(q, start, g, dir, i);
    }
    *start_out = start;
    return (int)err;
}

}  // extern "C"
