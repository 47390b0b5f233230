// tests/emu/ss_emu_dry_pool.cu - dry pools (ss_dry_pool, ss_dry_pick) on the CPU.
//
// TEST INFRASTRUCTURE: runs the head of k_blocks for a pooled slot of a device pool (pick_pooled of ss_phases.cuh: the
// trajectory pick, then the dry pick of a dry-picked slot) on a Source whose counts block is laid out as chunk_describe
// lays it out, and k_draw's choice of a speaker's level table (speaker_table) followed by the per-try functions k_draw
// runs in its lanes (draw_span, draw_start, draw_silent).  Built with g++ (`-x c++`) by tests/test_dry_pool.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// One pooled slot over a pool of n candidates (candidate i: N[i], P[i], K[i] partitions when parts != 0, else K; gains
// g[i] when gains != 0) whose dry picks come from a dry pool of n_dry signals (n_dry == 0: no dry pick).  The signals'
// and the candidates' x / spec / cut / bounds are distinct dummy addresses.  out[] receives: error bits, x (index of the
// dry signal it points at, or -1 - candidate index when it is a candidate's own x), N, P, K, nb, bounds (candidate
// index), spec (candidate index), cut (candidate index or -1), h_rows, gain.
int emu_pick_pooled(const int* N, const int* P, const int* Ks, int parts, const float* g, int gains, int n, int K,
                    int C, int direct, int n_dry, int pick, int dry_pick, double* out) {
    static float xs[64], drys[64];
    static int bnds[64], cuts[64];
    static float2 specs[64];
    PoolEntry table[64];
    const float* dtab[64];
    for (int i = 0; i < n; ++i) {
        table[i].x = xs + i; table[i].bounds = bnds + i; table[i].spec = specs + i; table[i].cut = cuts + i;
        table[i].N = N[i]; table[i].P = P[i];
    }
    for (int i = 0; i < n_dry; ++i) dtab[i] = drys + i;
    alignas(16) int counts[28];
    memset(counts, 0, sizeof(counts));
    Source s;
    memset(&s, 0, sizeof(s));
    s.C = C; s.K = K; s.mode = MODE_MOVING_BOUNDS;
    float dummy_out;
    s.out_direct = direct ? &dummy_out : nullptr;
    s.counts = counts;
    const PoolEntry* tp = table;
    const int* pick_p = &pick;
    const float* gp = gains ? g : nullptr;
    const int* kp = parts ? Ks : nullptr;
    memcpy(counts + 8, &tp, sizeof(tp));
    counts[10] = n;
    const float one = 1.0f;
    memcpy(counts + 11, &one, sizeof(one));
    memcpy(counts + 12, &pick_p, sizeof(pick_p));
    memcpy(counts + 14, &gp, sizeof(gp));
    memcpy(counts + 16, &kp, sizeof(kp));
    const int* dpick_p = &dry_pick;
    const float* const* dt = n_dry ? dtab : nullptr;
    memcpy(counts + 20, &dt, sizeof(dt));
    memcpy(counts + 22, &dpick_p, sizeof(dpick_p));
    counts[24] = n_dry;
    const unsigned err = pick_pooled(s);
    int xi = -1000;
    if (s.x >= drys && s.x < drys + 64) xi = (int)(s.x - drys);
    else if (s.x >= xs && s.x < xs + 64) xi = -1 - (int)(s.x - xs);
    out[0] = err; out[1] = xi; out[2] = s.N; out[3] = s.P; out[4] = s.K; out[5] = s.nb;
    out[6] = (double)(s.bounds - bnds); out[7] = (double)(s.hspec - specs); out[8] = s.cut ? (double)(s.cut - cuts) : -1;
    out[9] = s.h_rows; out[10] = stem_gain(s);
    return 0;
}

// One draw as k_draw makes it: reader r has a pool of cand_n[r] candidates whose N are at cand_N + cand_off[r] and whose
// level tables are cand_Q[cand_off[r] + i], picked by picks[r]; a speaker k (reader spk[k]) with dry_n[spk[k]] > 0 tests
// the dry table dry_Q[dry_off[spk[k]] + clamp(dry_picks[spk[k]])] with D = len, else its pool's table with D[k].
// Returns the start, *used the 1-based index of the kept try or 0.
int emu_draw_mixed(const int* cand_N, const double* const* cand_Q, const int* cand_off, const int* cand_n,
                   const int* picks, const double* const* dry_Q, const int* dry_off, const int* dry_n,
                   const int* dry_picks, int n_readers, const int* spk, const double* D, int S, int len, const double* u,
                   int tries, float threshold_db, int* used) {
    bool bad;
    int M = 0x7fffffff;
    for (int r = 0; r < n_readers; ++r) {
        const int m = draw_span(cand_N[cand_off[r] + clamp_pick(picks[r], cand_n[r], bad)], len);
        M = m < M ? m : M;
    }
    const double* Q[8];
    double Dk[8];
    for (int k = 0; k < S; ++k) {
        const int r = spk[k];
        const bool dry = dry_n[r] > 0;
        Q[k] = speaker_table(cand_Q + cand_off[r], picks + r, cand_n[r], dry ? dry_Q + dry_off[r] : nullptr,
                             dry_picks + r, dry_n[r]);
        Dk[k] = dry ? (double)len : D[k];
    }
    int s = 0;
    for (int t = 0; t < tries; ++t) {
        s = draw_start(u[t], M);
        bool silent = false;
        for (int k = 0; k < S; ++k) silent = silent || draw_silent(Q[k], s, len, Dk[k], threshold_db);
        if (!silent) { *used = t + 1; return s; }
    }
    *used = 0;
    return s;
}

}  // extern "C"
