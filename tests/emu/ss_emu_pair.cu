// tests/emu/ss_emu_pair.cu - pair gains (ss_pair_gains) in the heads of k_blocks and k_stage, on the CPU.
//
// TEST INFRASTRUCTURE: runs pick_pooled (the head of k_blocks for a pooled slot of a device pool) on a Source whose
// counts block is laid out as chunk_describe lays it out for a dry-picked slot, pair table included, and stage_head (the
// head of k_stage for a staged slot) on the same pool, picks and table.  Built with g++ (`-x c++`) by
// tests/test_pair_gains.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// One dry-picked slot over a static pool of n candidates of N[i] samples (pool gains g[i] when gains != 0) and a dry
// pool of n_dry signals, with the pair table tab (n_dry * n floats, pair (d, i) at [d * n + i]) when table != 0.
// out receives pick_pooled's error bits, stem gain and dry signal index (the signal x points at), then stage_head's
// error bits, view gain and dry signal index, for pick v and dry pick dv.
int emu_pair_heads(const int* N, const float* g, int gains, int n, int n_dry, const float* tab, int table, int v, int dv,
                   double* out) {
    static float xs[64], drys[64];
    static float2 specs[64];
    PoolEntry pool[64];
    const float* dtab[64];
    for (int i = 0; i < n; ++i) {
        pool[i].x = xs + i; pool[i].bounds = nullptr; pool[i].spec = specs + i; pool[i].cut = nullptr;
        pool[i].N = N[i]; pool[i].P = 1;
    }
    for (int i = 0; i < n_dry; ++i) dtab[i] = drys + i;
    const float* const gp = gains ? g : nullptr;
    const float* const tp = table ? tab : nullptr;
    // k_blocks: the 112-byte counts block of a dry-picked slot
    alignas(16) int counts[28];
    memset(counts, 0, sizeof(counts));
    Source s;
    memset(&s, 0, sizeof(s));
    s.C = 1; s.K = 1; s.mode = MODE_STATIC;
    s.counts = counts;
    const PoolEntry* pp = pool;
    const int* pick_p = &v;
    const int* dpick_p = &dv;
    const float* const* dt = dtab;
    memcpy(counts + 8, &pp, sizeof(pp));
    counts[10] = n;
    const float one = 1.0f;
    memcpy(counts + 11, &one, sizeof(one));
    memcpy(counts + 12, &pick_p, sizeof(pick_p));
    memcpy(counts + 14, &gp, sizeof(gp));
    memcpy(counts + 20, &dt, sizeof(dt));
    memcpy(counts + 22, &dpick_p, sizeof(dpick_p));
    counts[24] = n_dry;
    memcpy(counts + 26, &tp, sizeof(tp));
    out[0] = pick_pooled(s);
    out[1] = stem_gain(s);
    out[2] = (double)(s.x - drys);
    // k_stage: a slot of a device pool (no rows staged) whose dry pick comes from a host dry pool
    StageView view;
    const float* src = nullptr;
    int x0 = 0, x1 = 0;
    out[3] = stage_head(pool, n, v, nullptr, 1, gp, nullptr, 0, 1, 1, false, dtab, dv, n_dry, view, src, x0, x1, tp);
    out[4] = view.gain;
    out[5] = (double)(src - drys);
    return 0;
}

}  // extern "C"
