// tests/emu/ss_emu_layout.cu - layout draws of plans (ss_layout_draw) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE: runs what k_layout runs for one draw - the Philox4x32-10 generator and layout_row of
// ss_phases.cuh over the same scratch.  Built with g++ (`-x c++`) by tests/test_layout_draw.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// out[0..3] = philox4x32_10(ctr, key)
void emu_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
    const uint4 v = philox4x32_10(make_uint4(ctr[0], ctr[1], ctr[2], ctr[3]), key[0], key[1]);
    out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w;
}

// `count` uniform integers below k[i] from the word stream of draw r at (rng[0], rng[1]), in order
void emu_rng_below(const int64_t* rng, int r, const uint64_t* k, int count, uint64_t* out) {
    LayoutRng g = layout_rng(rng[0], rng[1], r);
    for (int i = 0; i < count; ++i) out[i] = rng_below(g, k[i]);
}

// `rows` rows of layout draw r, row q at (rng[2q], rng[2q + 1]), over n clips of `lengths` (select: a bed's selection
// lengths or null) with bound K, as k_layout draws them: streams with heads == null, else beds.  Each array receives
// rows * m entries, row after row.
void emu_layout_rows(const int64_t* rng, int rows, int r, const int* lengths, const int* select, int n, int m, int total,
                     int gap_max, int K, int* ids, int* offsets, int* heads, int* counts) {
    LayoutDesc d;
    memset(&d, 0, sizeof(d));
    d.lengths = lengths; d.select = select; d.n = n; d.m = m; d.total = total; d.gap_max = gap_max; d.K = K; d.r = r;
    d.map_cap = layout_map_cap(K);
    std::vector<int> s(layout_scratch_ints(K));
    for (int q = 0; q < rows; ++q) {
        const size_t o = (size_t)q * m;
        d.rng = rng + 2 * q; d.ids = ids + o; d.offsets = offsets + o;
        d.heads = heads ? heads + o : nullptr; d.counts = counts ? counts + o : nullptr;
        for (int i = 0; i < d.map_cap; ++i) s[i] = -1;
        layout_row(d, s.data(), s.data() + d.map_cap, s.data() + 2 * d.map_cap);
    }
}

// The walk of k_stage and k_draw (stream_entries with heads == null, else bg_entries) over one row: the error bits;
// *kept receives the number of kept entries
int emu_layout_walk(const int* ids, const int* offsets, const int* heads, const int* counts, int m, const int* lengths,
                    int n, int* kept) {
    int k = 0;
    auto len = [&](int, int id) { return lengths[id]; };
    const unsigned err = heads ? bg_entries(ids, offsets, heads, counts, m, n, len,
                                            [&](int, int, int, int, int) { ++k; return true; })
                               : stream_entries(ids, offsets, m, n, len, [&](int, int, int, int) { ++k; return true; });
    *kept = k;
    return (int)err;
}

}  // extern "C"
