// tests/emu/ss_emu_stage.cu - host pools in the emulated kernels: a pooled slot staged by k_stage's read set.
//
// TEST INFRASTRUCTURE, like ss_emu_pool_lengths.cu, whose bank builder and emulated phases it reuses (included below).
// Exports one pooled slot run twice through the head of k_blocks, the rest of the block table, k_prepare's dry windows
// and range warps and the render CTAs: over the full candidate (pick_slot of a device pool) and over a staged view
// (take_view) whose x and spectra hold only the read set (stage_set) - every other sample and row is NaN, so a read
// outside the set shows in the output.  Also exports stage_set and stage_cap.  Built with g++ (`-x c++`) by
// tests/test_host_pool.py.
#include "ss_emu_bank.cu"

#include <cmath>

namespace {

// What one run of a slot produced: the Source after the head of k_blocks, its block table and work items, the output
struct SlotRun {
    Source S;
    int counts[20];
    std::vector<Block> blocks;
    std::vector<double> rstep;
    std::vector<float2> xs;
    std::vector<RItem> items;
    int n_items;
};

// The rest of k_blocks after its head (the host planner of the same table: window_blocks over the full plan), then
// k_prepare's range warps and, with `render`, its dry windows and the render CTAs of the kernel variant of the slot's K
// and blocking
void run_slot(SlotRun& R, int ws, int wl, int k_pool, bool render) {
    const Tables& T = tables();
    Source& S = R.S;
    const int cap = table_cap(S.aligned, S.nb, S.P);
    std::vector<Block> full((size_t)cap);
    const int nfull = plan_blocks(S.aligned, S.bounds, S.P, S.N, S.nb, 0, cap, full.data());
    const WinSpan w = window_blocks(full.data(), nfull < cap ? nfull : cap, ws, ws + wl, S.K);
    S.nblk_max = w.g1 - w.g0;
    R.blocks.assign((size_t)S.nblk_max, Block());
    const int nplan = plan_blocks(S.aligned, S.bounds, S.P, S.N, S.nb, w.g0, w.g1, R.blocks.data());
    const int nblk = (nplan < w.g1 ? nplan : w.g1) - w.g0;
    clear_blocks(R.blocks.data(), nblk, S.nblk_max, 0, 1);
    R.rstep.assign((size_t)S.P, 0.0);
    if (S.mode == MODE_MOVING_BOUNDS) fill_rstep(S.bounds, S.P, R.rstep.data(), 0, 1);
    R.counts[0] = nblk; R.counts[1] = 0; R.counts[2] = w.k0 - w.g0; R.counts[3] = w.k1 - w.k0;
    R.counts[4] = ws; R.counts[5] = wl;
    S.blocks = R.blocks.data(); S.rstep = R.rstep.data();
    R.xs.assign((size_t)S.nblk_max * kSpec, float2());
    S.xspec = R.xs.data();
    R.items.assign((size_t)max_render_items(S), RItem());
    for (int i = 0; render && i < spectra_pairs_x(S); ++i) cta_spectra(S, i, T);
    prepare_ranges(S, R.items.data());
    R.n_items = win_blocks(S) * items_per_block(S);
    if (!render) return;
    const int grid = R.n_items < 3 ? R.n_items : 3;
    for (int cta = 0; cta < grid; ++cta) {
        if (k_pool == 1 && one_transform_per_item(S.aligned, S.mode, S.K)) cta_render_fast(R.items.data(), R.n_items, cta, grid, T);
        else cta_render(R.items.data(), R.n_items, cta, grid, T, false, k_pool > 1);
    }
}

// a slot's Source before the head of k_blocks: the pool's shape, the slot's outputs and window
void slot_source(SlotRun& R, int C, int K, int mode, int aligned, int wl, float* out, float* out_direct) {
    memset(&R.S, 0, sizeof(R.S));
    memset(R.counts, 0, sizeof(R.counts));
    R.S.C = C; R.S.K = K; R.S.mode = mode; R.S.aligned = aligned; R.S.out = out; R.S.out_direct = out_direct;
    R.counts[5] = wl;
    R.S.counts = R.counts;
}

}  // namespace

extern "C" {

// stage_set: out = [xa, xb, row0, rows]
int emu_stage_set(int N, int P, int C, int K, const int32_t* bounds, int ws, int len, int* out) {
    const StageSet r = stage_set(N, P, C, K, bounds, ws, len);
    out[0] = r.xa; out[1] = r.xb; out[2] = r.row0; out[3] = r.rows;
    return 0;
}

// stage_cap over n candidates (bounds == null: a static pool; candidate i's bounds at bounds + off[i]): out = [rows, nx]
int emu_stage_cap(const int32_t* bounds, const int64_t* off, const int* N, const int* P, const int* K, int n, int C,
                  int len, int* out) {
    std::vector<const int*> b;
    for (int i = 0; bounds && i < n; ++i) b.push_back(bounds + off[i]);
    stage_cap(bounds ? b.data() : nullptr, N, P, K, n, C, len, out[0], out[1]);
    return 0;
}

// One pooled slot over a candidate (x: N samples; spec / cut: its bank, with a direct set when direct != 0) in a pool of
// K_pool partitions (the kernel variant) and the given blocking, at window [ws, ws + wl): rendered over the full
// candidate into out_full (and outd_full) and over the staged view into out_staged (and outd_staged) - without `render`
// only the tables and items are built.  info receives
//   [0..3]   stage_set: xa, xb, row0, rows
//   [4..7]   what the render reads, from the block table: the least and largest dry sample + 1 of the table's blocks'
//            windows, and window_rows of the positions of the blocks that meet the window: row0, rows
//   [8]      1 if both runs built the same Source fields (x and spectra through their origins), block table and items
//   [9..12]  h_row0, h_rows of the full run and of the staged run
//   [13..14] the direct set's offset in rows (rows_stored_h) of the full run and of the staged run, or -1 without one
int emu_stage_slot(const float* x, const float2* spec, const int* cut, const int32_t* bounds, int N, int P, int C,
                   int L, int mode, int aligned, int K_pool, int ws, int wl, int direct, int render, float* out_full,
                   float* out_staged, float* outd_full, float* outd_staged, int* info) {
    const int K = (L + kB - 1) / kB;
    const StageSet r = stage_set(N, P, C, K, bounds, ws, wl);
    info[0] = r.xa; info[1] = r.xb; info[2] = r.row0; info[3] = r.rows;
    // the staged copies: the read set and nothing else
    const float nanf_ = std::nanf("");
    std::vector<float> xs((size_t)(r.xb - r.xa) + 1, nanf_);
    for (int n = r.xa; n < r.xb; ++n) xs[(size_t)(n - r.xa)] = x[n];
    const int sets = direct ? 2 : 1;
    const size_t rows_h = (size_t)P * C * K;
    std::vector<float2> ss((size_t)sets * r.rows * kSpec);
    for (int s = 0; s < sets; ++s)
        memcpy(ss.data() + (size_t)s * r.rows * kSpec, spec + (s * rows_h + r.row0) * kSpec,
               sizeof(float2) * (size_t)r.rows * kSpec);
    // full: a device pool of one candidate, pick_parts + pick_slot
    PoolEntry e;
    e.x = x; e.bounds = mode == MODE_MOVING_BOUNDS ? bounds : nullptr; e.spec = const_cast<float2*>(spec);
    e.cut = direct ? const_cast<int*>(cut) : nullptr; e.N = N; e.P = P;
    SlotRun F;
    slot_source(F, C, K_pool, mode, aligned, wl, out_full, direct ? outd_full : nullptr);
    const PoolEntry* table = &e;
    memcpy(F.counts + 8, &table, sizeof(table));
    F.counts[10] = 1;
    const int pick = 0, *pick_p = &pick, parts = K, *parts_p = &parts;
    memcpy(F.counts + 12, &pick_p, sizeof(pick_p));
    memcpy(F.counts + 16, &parts_p, sizeof(parts_p));
    bool bad = false;
    pick_parts(F.S, *pick_ptr(F.S));
    pick_slot(F.S, *pick_ptr(F.S), bad);
    // staged: the view k_stage writes, taken by the head of k_blocks
    StageView v;
    v.e = e; v.e.x = xs.data() - r.xa; v.e.spec = ss.data(); v.K = K; v.row0 = r.row0; v.rows = r.rows; v.gain = 1.0f;
    SlotRun G;
    slot_source(G, C, K_pool, mode, aligned, wl, out_staged, direct ? outd_staged : nullptr);
    const StageView* vp = &v;
    memcpy(G.counts + 8, &table, sizeof(table));
    memcpy(G.counts + 18, &vp, sizeof(vp));
    take_view(G.S, *stage_view(G.S));
    run_slot(F, ws, wl, K_pool, render != 0);
    run_slot(G, ws, wl, K_pool, render != 0);
    // what the render read, from the full run's table
    int xa = N, xb = 0, pa = P, pb = -1;
    for (int b = 0; b < F.counts[0]; ++b) {
        const Block& bk = F.blocks[(size_t)b];
        const int a0 = bk.start - kB > 0 ? bk.start - kB : 0, b0 = bk.start + kB < N ? bk.start + kB : N;
        xa = a0 < xa ? a0 : xa; xb = b0 > xb ? b0 : xb;
        if ((unsigned)(b - win_first(F.S)) < (unsigned)win_blocks(F.S)) {
            const Block q = block_positions(F.S, bk, 0, 0);
            pa = q.p_lo < pa ? q.p_lo : pa; pb = q.p_hi > pb ? q.p_hi : pb;
        }
    }
    info[4] = xa; info[5] = xb;
    window_rows(P, C, K, pa, pb, info[6], info[7]);
    // the same Source, tables and items through each run's origins
    bool same = F.S.N == G.S.N && F.S.P == G.S.P && F.S.K == G.S.K && F.S.nb == G.S.nb && F.S.bounds == G.S.bounds &&
                F.S.cut == G.S.cut && F.S.x - x == G.S.x - (xs.data() - r.xa) && F.counts[0] == G.counts[0] &&
                F.counts[2] == G.counts[2] && F.counts[3] == G.counts[3] && F.n_items == G.n_items &&
                stem_gain(F.S) == stem_gain(G.S);
    for (int b = 0; same && b < F.counts[0]; ++b) {
        const Block& p = F.blocks[(size_t)b], &q = G.blocks[(size_t)b];
        same = p.start == q.start && p.len == q.len && p.p_lo == q.p_lo && p.p_hi == q.p_hi;
    }
    // the row of the bank an item's H0 names: through its set's offset (rows_stored_h) and the row origin h_row0
    const int per = items_per_set(F.S), ipb = items_per_block(F.S);
    auto row_of = [&](const SlotRun& R, const float2* base, int i) {
        const int set = i % ipb >= per ? 1 : 0;
        return (long long)(R.items[(size_t)i].H0 - base) / kSpec - (long long)set * rows_stored_h(R.S) + R.S.h_row0;
    };
    for (int i = 0; same && i < F.n_items; ++i) {
        const RItem& p = F.items[(size_t)i], &q = G.items[(size_t)i];
        same = p.X - F.xs.data() == q.X - G.xs.data() && row_of(F, spec, i) == row_of(G, ss.data(), i) &&
               p.row - (i % ipb >= per ? outd_full : out_full) == q.row - (i % ipb >= per ? outd_staged : out_staged) &&
               (p.row1 == nullptr) == (q.row1 == nullptr) && p.pstride == q.pstride && p.n0 == q.n0 &&
               p.n_end == q.n_end && p.n_lo == q.n_lo && p.p_lo == q.p_lo && p.p_hi == q.p_hi && p.kparts == q.kparts &&
               p.mode == q.mode && p.gain == q.gain && p.b0 == q.b0 && p.step == q.step;
    }
    info[8] = same ? 1 : 0;
    info[9] = F.S.h_row0; info[10] = F.S.h_rows; info[11] = G.S.h_row0; info[12] = G.S.h_rows;
    info[13] = direct ? rows_stored_h(F.S) : -1;
    info[14] = direct ? rows_stored_h(G.S) : -1;
    return 0;
}

}  // extern "C"
