// tests/emu/ss_emu_layout_group.cu - grouped layout draws of plans (ss_layout_group) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE: runs what k_layout_grouped runs for one draw - layout_row_grouped of ss_phases.cuh over the same
// scratch.  Built with g++ (`-x c++`) by tests/group_reference.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// `rows` stream rows of layout draw r, row q at (rng[2q], rng[2q + 1]) over the group group[q] of the G groups that
// bounds (G + 1 entries) cut the n utterances of `lengths` into, with bound K, as k_layout_grouped draws them; bounds
// null: ungrouped rows (group is not read).  ids and offsets receive rows * m entries, row after row; the return value
// is the error bits of every row or-ed together.
int emu_layout_group_rows(const int64_t* rng, int rows, int r, const int* lengths, int n, int m, int total, int gap_max,
                          int K, const int* bounds, int G, const int* group, int* ids, int* offsets) {
    LayoutDesc d;
    memset(&d, 0, sizeof(d));
    d.lengths = lengths; d.n = n; d.m = m; d.total = total; d.gap_max = gap_max; d.K = K; d.r = r;
    d.map_cap = layout_map_cap(K);
    std::vector<int> s(layout_scratch_ints(K));
    unsigned err = 0;
    for (int q = 0; q < rows; ++q) {
        const size_t o = (size_t)q * m;
        d.rng = rng + 2 * q; d.ids = ids + o; d.offsets = offsets + o;
        LayoutGroup e;
        memset(&e, 0, sizeof(e));
        if (bounds) { e.group = group + q; e.bounds = bounds; e.G = G; }
        for (int i = 0; i < d.map_cap; ++i) s[i] = -1;
        err |= layout_row_grouped(d, e, s.data(), s.data() + d.map_cap, s.data() + 2 * d.map_cap);
    }
    return (int)err;
}

}  // extern "C"
