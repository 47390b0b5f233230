// tests/emu/ss_emu_stream.cu - dry streams (ss_dry_stream) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE: runs what k_stage<true, TAPS, true> and k_draw<true, true> run for a stream slot - the layout
// walk (stream_entries), its resolution into kept entries cut at the stream's length (stream_resolve), the per-sample
// staging (stream_sample) over the read set of k_stage's head (stage_head) and the per-utterance crop energies of the
// draws (draw_silent_stream).  Built with g++ (`-x c++`) by tests/test_dry_streams.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// The walk over m entries of a layout over n utterances of `lengths`: the kept entries' ids, offsets and lengths in
// order into kid / koff / klen, their count into *count.  Returns the error bits (kStreamBit for an invalid entry).
int emu_stream_walk(const int* ids, const int* offsets, int m, const int* lengths, int n, int* kid, int* koff,
                    int* klen, int* count) {
    int k = 0;
    const unsigned err = stream_entries(ids, offsets, m, n, [&](int, int id) { return lengths[id]; },
                                        [&](int, int id, int o, int l) {
                                            kid[k] = id; koff[k] = o; klen[k] = l; ++k;
                                            return true;
                                        });
    *count = k;
    return (int)err;
}

// k_stage for a stream slot of a device pool (one candidate of N samples, P positions, bounds, K partitions) at window
// [ws, ws + wl): the head (stage_head, no dry table), then the layout loaded per entry as the CTA loads it, resolved at
// `cut` and staged sample by sample into out (x1 - x0 floats).  info receives [0..1] x0, x1, [2] 1 if the view is the
// one a dry-picked slot of the same candidate gets.  Returns the error bits of the head and of the walk.
int emu_stream_stage(const int32_t* bounds, int N, int P, int C, int K, int ws, int wl, const int* ids,
                     const int* offsets, int m, const int* lengths, const int16_t* const* sig, int n, int cut,
                     float* out, int* info) {
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
    std::vector<const int16_t*> s(m), p(m);
    for (int j = 0; j < m; ++j) {
        const bool ok = ids[j] >= 0 && ids[j] < n;
        len[j] = ok ? lengths[ids[j]] : 0;
        s[j] = ok ? sig[ids[j]] : nullptr;
    }
    int k;
    err |= stream_resolve(ids, offsets, len.data(), s.data(), m, n, cut, a.data(), b.data(), p.data(), &k);
    for (int t = 0; t < x1 - x0; ++t) out[t] = stream_sample(a.data(), b.data(), p.data(), k, x0 + t);
    return (int)err;
}

// One draw as k_draw<true, true> makes it for a single stream speaker over a 16-bit pool of n utterances (signals sig,
// sparse tables levels): M the draw's span.  Returns the start, *used the 1-based index of the kept try or 0.
int emu_draw_stream(const int* ids, const int* offsets, int m, const int* lengths, const int16_t* const* sig,
                    const double* const* levels, int n, int cut, int M, int len, const double* u, int tries,
                    float threshold_db, int* used) {
    const DryStream d = {ids, offsets, lengths, sig, levels, m, n, cut, 0};
    int s = 0;
    for (int t = 0; t < tries; ++t) {
        s = draw_start(u[t], M);
        if (!draw_silent_stream(d, s, len, threshold_db)) { *used = t + 1; return s; }
    }
    *used = 0;
    return s;
}

}  // extern "C"
