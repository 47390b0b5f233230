// tests/emu/ss_emu_dry_stage.cu - host dry pools in the emulated kernels: a dry-picked slot of a device pool whose dry
// samples k_stage stages.
//
// TEST INFRASTRUCTURE, like ss_emu_stage.cu, whose slot runner, bank builder and emulated phases it reuses (included
// below).  Exports one pooled slot of a device pool with a dry pick, run twice through the head of k_blocks, the rest of
// the block table, k_prepare's dry windows and range warps and the render CTAs: with the dry pick made by k_blocks
// (pick_pooled, a device dry pool) and with the view k_stage writes (stage_head, then take_view), whose x is a staging
// copy of the picked signal's whole float4s [xa & ~3, (xb + 3) & ~3) as a host dry pool's arena holds them (zero-padded
// past the signal's end) and NaN everywhere else, so a read outside the staged span shows in the output.  Built with g++
// (`-x c++`) by tests/test_host_dry_pool.py.
#include "ss_emu_stage.cu"

extern "C" {

// One dry-picked slot over a candidate (spec / cut: its bank, with a direct set when direct != 0; N samples, its own x is
// never read) in a pool of K_pool partitions (the kernel variant) and the given blocking, at window [ws, ws + wl), with
// dry pick `dv` into a dry pool of n_dry copies of the signal d (Nd >= N samples): rendered with the pick of k_blocks into
// out_dev (and outd_dev) and over k_stage's staged view into out_staged (and outd_staged) - without `render` only the
// tables and items are built.  info receives
//   [0..1]   the staged span x0, x1 (whole float4s), [2..3] stage_set's xa, xb
//   [4..5]   what the render reads, from the block table: the least and largest dry sample + 1 of the table's blocks' windows
//   [6]      1 if both runs built the same Source fields (x through its origin), block table and items
//   [7..10]  h_row0, h_rows of the k_blocks run and of the staged run
//   [11..12] the direct set's offset in rows (rows_stored_h) of both runs, or -1 without one
//   [13..14] the error bits of pick_pooled and of stage_head
//   [15]     1 if the staged view keeps the bank's spectra and the candidate's bounds, N, P, K and gain
int emu_dry_stage_slot(const float* cx, const float2* spec, const int* cut, const int32_t* bounds, int N, int P, int C,
                       int L, int mode, int aligned, int K_pool, int ws, int wl, int direct, const float* d, int Nd,
                       int n_dry, int dv, int render, float* out_dev, float* out_staged, float* outd_dev,
                       float* outd_staged, int* info) {
    const int K = (L + kB - 1) / kB;
    PoolEntry e;
    e.x = cx; e.bounds = mode == MODE_MOVING_BOUNDS ? bounds : nullptr; e.spec = const_cast<float2*>(spec);
    e.cut = direct ? const_cast<int*>(cut) : nullptr; e.N = N; e.P = P;
    const PoolEntry* table = &e;
    const int pick = 0, *pick_p = &pick, parts = K, *parts_p = &parts;
    // the dry pool: n_dry signals, every one the arena's copy of d (zero-padded to whole float4s)
    std::vector<float> arena((size_t)((Nd + 3) & ~3), 0.0f);
    memcpy(arena.data(), d, sizeof(float) * (size_t)Nd);
    std::vector<const float*> dtab((size_t)n_dry, arena.data());
    const float* const* dt = dtab.data();
    // k_blocks: a device pool of one candidate with a device dry pool (pick_pooled)
    SlotRun F;
    slot_source(F, C, K_pool, mode, aligned, wl, out_dev, direct ? outd_dev : nullptr);
    memcpy(F.counts + 8, &table, sizeof(table));
    F.counts[10] = 1;
    memcpy(F.counts + 12, &pick_p, sizeof(pick_p));
    memcpy(F.counts + 16, &parts_p, sizeof(parts_p));
    int counts_dry[28];                                  // the 112-byte counts block of a dry-picked slot
    memset(counts_dry, 0, sizeof(counts_dry));
    memcpy(counts_dry, F.counts, sizeof(F.counts));
    const int* dpick_p = &dv;
    memcpy(counts_dry + 20, &dt, sizeof(dt));
    memcpy(counts_dry + 22, &dpick_p, sizeof(dpick_p));
    counts_dry[24] = n_dry;
    F.S.counts = counts_dry;
    info[13] = (int)pick_pooled(F.S);
    memcpy(F.counts, counts_dry, sizeof(F.counts));
    F.S.counts = F.counts;
    // k_stage: the head, then the staged copy of [x0, x1) and the view the head of k_blocks takes (take_view)
    StageView v;
    const float* src = nullptr;
    int x0 = 0, x1 = 0;
    info[14] = (int)stage_head(&e, 1, pick, parts_p, K_pool, nullptr, nullptr, ws, wl, C, false, dt, dv, n_dry, v, src,
                               x0, x1);
    const StageSet r = stage_set(N, P, C, K, e.bounds, ws, wl);
    info[0] = x0; info[1] = x1; info[2] = r.xa; info[3] = r.xb;
    const float nanf_ = std::nanf("");
    std::vector<float> xs((size_t)(x1 - x0) + 8, nanf_);          // NaN behind the staged span
    for (int n = x0; n < x1; ++n) xs[(size_t)(n - x0)] = src[n];
    info[15] = v.e.spec == e.spec && v.e.bounds == e.bounds && v.e.cut == e.cut && v.e.N == N && v.e.P == P &&
               v.K == K && v.gain == 1.0f;
    v.e.x = xs.data() - x0;
    SlotRun G;
    slot_source(G, C, K_pool, mode, aligned, wl, out_staged, direct ? outd_staged : nullptr);
    const StageView* vp = &v;
    memcpy(G.counts + 8, &table, sizeof(table));
    memcpy(G.counts + 18, &vp, sizeof(vp));
    take_view(G.S, *stage_view(G.S));
    run_slot(F, ws, wl, K_pool, render != 0);
    run_slot(G, ws, wl, K_pool, render != 0);
    int xa = N, xb = 0;
    for (int b = 0; b < F.counts[0]; ++b) {
        const Block& bk = F.blocks[(size_t)b];
        const int a0 = bk.start - kB > 0 ? bk.start - kB : 0, b0 = bk.start + kB < N ? bk.start + kB : N;
        xa = a0 < xa ? a0 : xa; xb = b0 > xb ? b0 : xb;
    }
    info[4] = xa; info[5] = xb;
    bool same = F.S.N == G.S.N && F.S.P == G.S.P && F.S.K == G.S.K && F.S.nb == G.S.nb && F.S.bounds == G.S.bounds &&
                F.S.cut == G.S.cut && F.S.hspec == G.S.hspec && F.S.x - arena.data() == G.S.x - (xs.data() - x0) &&
                F.counts[0] == G.counts[0] && F.counts[2] == G.counts[2] && F.counts[3] == G.counts[3] &&
                F.n_items == G.n_items && stem_gain(F.S) == stem_gain(G.S);
    for (int b = 0; same && b < F.counts[0]; ++b) {
        const Block& p = F.blocks[(size_t)b], &q = G.blocks[(size_t)b];
        same = p.start == q.start && p.len == q.len && p.p_lo == q.p_lo && p.p_hi == q.p_hi;
    }
    const int per = items_per_set(F.S), ipb = items_per_block(F.S);
    for (int i = 0; same && i < F.n_items; ++i) {
        const RItem& p = F.items[(size_t)i], &q = G.items[(size_t)i];
        same = p.X - F.xs.data() == q.X - G.xs.data() && p.H0 == q.H0 &&
               p.row - (i % ipb >= per ? outd_dev : out_dev) == q.row - (i % ipb >= per ? outd_staged : out_staged) &&
               (p.row1 == nullptr) == (q.row1 == nullptr) && p.pstride == q.pstride && p.n0 == q.n0 &&
               p.n_end == q.n_end && p.n_lo == q.n_lo && p.p_lo == q.p_lo && p.p_hi == q.p_hi && p.kparts == q.kparts &&
               p.mode == q.mode && p.gain == q.gain && p.b0 == q.b0 && p.step == q.step;
    }
    info[6] = same ? 1 : 0;
    info[7] = F.S.h_row0; info[8] = F.S.h_rows; info[9] = G.S.h_row0; info[10] = G.S.h_rows;
    info[11] = direct ? rows_stored_h(F.S) : -1;
    info[12] = direct ? rows_stored_h(G.S) : -1;
    return 0;
}

}  // extern "C"
