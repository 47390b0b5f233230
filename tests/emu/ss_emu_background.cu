// tests/emu/ss_emu_background.cu - background streams (ss_bg_stream) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE: runs what k_stage<true, TAPS, true, true> runs for a bed slot - the layout walk (bg_entries), its
// resolution into kept entries cut at the stream's length (bg_resolve) and the per-sample staging (bg_sample) over the
// read set of k_stage's head (stage_head), for int16 and float32 clips.  Built with g++ (`-x c++`) by
// tests/test_background_streams.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// The walk over m entries of a bed layout over n clips of `lengths`: the kept entries' ids, offsets, heads and counts
// in order into kid / koff / khead / kcnt, their count into *count.  Returns the error bits (kStreamBit for an invalid
// entry).
int emu_bg_walk(const int* ids, const int* offsets, const int* heads, const int* counts, int m, const int* lengths,
                int n, int* kid, int* koff, int* khead, int* kcnt, int* count) {
    int k = 0;
    const unsigned err = bg_entries(ids, offsets, heads, counts, m, n, [&](int, int id) { return lengths[id]; },
                                    [&](int, int id, int o, int h, int c) {
                                        kid[k] = id; koff[k] = o; khead[k] = h; kcnt[k] = c; ++k;
                                        return true;
                                    });
    *count = k;
    return (int)err;
}

// k_stage for a bed slot of a device pool (one candidate of N samples, P positions, bounds, K partitions) at window
// [ws, ws + wl): the head (stage_head, no dry table), then the layout loaded per entry as the CTA loads it, resolved at
// `cut` and staged sample by sample into out (x1 - x0 floats).  sig holds the n clips' addresses, int16 with i16 != 0,
// else float32.  info receives [0..1] x0, x1, [2] 1 if the view is the one a dry-picked slot of the same candidate
// gets.  Returns the error bits of the head and of the walk.
int emu_bg_stage(const int32_t* bounds, int N, int P, int C, int K, int ws, int wl, const int* ids, const int* offsets,
                 const int* heads, const int* counts, int m, const int* lengths, const char* const* sig, int i16, int n,
                 int cut, float* out, int* info) {
    PoolEntry e;
    memset(&e, 0, sizeof(e));
    e.bounds = P > 1 ? bounds : nullptr; e.N = N; e.P = P;
    StageView v, vd;
    const float* src = nullptr;
    int x0, x1, d0, d1;
    unsigned err = stage_head(&e, 1, 0, nullptr, K, nullptr, nullptr, ws, wl, C, false, nullptr, 0, 0, v, src, x0, x1);
    const float* one = nullptr;
    stage_head(&e, 1, 0, nullptr, K, nullptr, nullptr, ws, wl, C, false, &one, 0, 1, vd, src, d0, d1);
    info[0] = x0; info[1] = x1;
    info[2] = memcmp(&v, &vd, sizeof(StageView)) == 0 && d0 == x0 && d1 == x1;
    std::vector<int> len(m), a(m), b(m);
    std::vector<const char*> s(m), p(m);
    for (int j = 0; j < m; ++j) {
        const bool ok = ids[j] >= 0 && ids[j] < n;
        len[j] = ok ? lengths[ids[j]] : 0;
        s[j] = ok ? sig[ids[j]] : nullptr;
    }
    int k;
    err |= bg_resolve(ids, offsets, heads, counts, len.data(), s.data(), i16 ? 2 : 4, m, n, cut, a.data(), b.data(),
                      p.data(), &k);
    for (int t = 0; t < x1 - x0; ++t) out[t] = bg_sample(a.data(), b.data(), p.data(), k, x0 + t, i16 != 0);
    return (int)err;
}

}  // extern "C"
