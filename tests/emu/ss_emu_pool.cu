// tests/emu/ss_emu_pool.cu - the planning helpers of a pooled slot (ss_source.pool + pick_dev) on the CPU.
//
// TEST INFRASTRUCTURE: exports the functions of ss_phases.cuh that size a pooled slot's block table (pool_table_cap,
// over the candidates' full plans under the pool's blocking), clamp a pick read from device memory (clamp_pick, as
// k_blocks does) and write the picked candidate into a slot's Source (pick_candidate).  Built with g++ (`-x c++`) by
// tests/test_pool.py.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// Table size of a pooled slot with windows of win_len: n candidates, candidate i with N[i], P[i] and (moving pool) its
// bounds at bounds[off[i]]; bounds == null for a static pool.
int emu_pool_table_cap(const int32_t* bounds, const int64_t* off, const int* N, const int* P, int n, int aligned,
                       int L, int win_len) {
    std::vector<const int*> b;
    int cap = 0;
    for (int i = 0; i < n; ++i) {
        if (bounds) b.push_back(bounds + off[i]);
        const int c = table_cap(aligned, (N[i] + kB - 1) / kB, P[i]);
        cap = c > cap ? c : cap;
    }
    std::vector<Block> full((size_t)cap);
    return pool_table_cap(aligned, bounds ? b.data() : nullptr, N, P, n, win_len, (L + kB - 1) / kB, full.data());
}

// k_blocks' clamp of a pick read from device memory; *bad = 1 when it was outside [0, n)
int emu_clamp_pick(int v, int n, int* bad) {
    bool b = false;
    const int r = clamp_pick(v, n, b);
    *bad = b ? 1 : 0;
    return r;
}

// pick_candidate on a slot of C channels, K partitions, with or without a direct output: out[] receives
// N, P, nb, h_row0, h_rows, and whether x, bounds, hspec and cut took the entry's pointers
int emu_pick_candidate(int N, int P, int C, int K, int direct, int* out) {
    Source s;
    memset(&s, 0, sizeof(s));
    s.C = C; s.K = K;
    float dummy_out;
    s.out_direct = direct ? &dummy_out : nullptr;
    static float x[1];
    static int bounds[1], cut[1];
    static float2 spec[1];
    PoolEntry e;
    e.x = x; e.bounds = bounds; e.spec = spec; e.cut = cut; e.N = N; e.P = P;
    pick_candidate(s, e);
    out[0] = s.N; out[1] = s.P; out[2] = s.nb; out[3] = s.h_row0; out[4] = s.h_rows;
    out[5] = s.x == x; out[6] = s.bounds == bounds; out[7] = s.hspec == spec; out[8] = s.cut == cut;
    out[9] = s.rir == nullptr && s.norm_part == nullptr;
    return 0;
}

}  // extern "C"
