// tests/emu/ss_emu_pool_lengths.cu - pools whose candidates differ in L, in the emulated kernels.
//
// TEST INFRASTRUCTURE, like ss_emu_bank.cu, whose bank builder and emulated phases it reuses (included below).  Exports
// the head of k_blocks for a slot over a pool whose candidates differ in K (pick_parts, then pick_slot) together with the
// work items fill_items then writes, pool_table_cap with each candidate's own K, and a banked windowed source rendered
// as a pooled slot renders it: grid blocking and, on request, k_render<LONG> whatever the source's own K.  Built with
// g++ (`-x c++`) by tests/test_pool_lengths.py.
#include "ss_emu_bank.cu"

extern "C" {

// A slot of C channels over a moving pool of n candidates (candidate i: N[i], P[i], K[i] partitions, its own spectra and
// cuts), pool K K_pool and parts = K (or null: a uniform pool), picks v: k_blocks' pick_parts + pick_slot, then the items
// fill_items writes for the block starting at 4096 * blk (a direct-target slot when direct != 0).  out receives
// [picked index, K, N, P, nb, h_rows, rows_stored_h, kparts, pstride / 4096, channel stride / 4096, direct H0 offset / 4096
// (0 without a direct set), bad]
int emu_pick_parts(int v, int n, const int* N, const int* P, const int* K, int uniform, int K_pool, int C, int direct,
                   int blk, int* out) {
    std::vector<PoolEntry> pool((size_t)n);
    static float x[1];
    static int bounds[1], cut[1];
    std::vector<float2> spec((size_t)n);
    for (int i = 0; i < n; ++i) {
        pool[i].x = x; pool[i].bounds = bounds; pool[i].spec = spec.data() + i; pool[i].cut = cut;
        pool[i].N = N[i]; pool[i].P = P[i];
    }
    int counts[20] = {};
    const PoolEntry* table = pool.data();
    memcpy(counts + 8, &table, sizeof(table));
    counts[10] = n;
    const int* pick = &v;
    memcpy(counts + 12, &pick, sizeof(pick));
    const int* parts = uniform ? nullptr : K;
    memcpy(counts + 16, &parts, sizeof(parts));
    Source s;
    memset(&s, 0, sizeof(s));
    float row[1];
    s.C = C; s.K = K_pool; s.mode = MODE_MOVING_BOUNDS; s.counts = counts; s.out = row;
    s.out_direct = direct ? row : nullptr;
    bool bad = false;
    pick_parts(s, *pick_ptr(s));
    pick_slot(s, *pick_ptr(s), bad);
    std::vector<RItem> items((size_t)items_per_block(s));
    Block bk; bk.start = kB * blk; bk.len = kB; bk.p_lo = 0; bk.p_hi = 1;
    fill_items(s, items.data(), 0, bk, 0, 1);
    const float2* spec0 = s.hspec;
    out[0] = (int)(s.hspec - spec.data()); out[1] = s.K; out[2] = s.N; out[3] = s.P; out[4] = s.nb; out[5] = s.h_rows;
    out[6] = rows_stored_h(s); out[7] = items[0].kparts; out[8] = items[0].pstride / kSpec;
    out[9] = C > 1 ? (int)((items[1].H0 - items[0].H0) / kSpec) : 0;
    out[10] = direct ? (int)((items[C].H0 - spec0) / kSpec) : 0;
    out[11] = bad ? 1 : 0;
    return 0;
}

// pool_table_cap with candidate i's own K[i] (bounds == null: a static pool)
int emu_pool_table_cap_parts(const int32_t* bounds, const int64_t* off, const int* N, const int* P, const int* K, int n,
                             int aligned, int win_len) {
    std::vector<const int*> b;
    int cap = 0, k_max = 0;
    for (int i = 0; i < n; ++i) {
        if (bounds) b.push_back(bounds + off[i]);
        const int c = table_cap(aligned, (N[i] + kB - 1) / kB, P[i]);
        cap = c > cap ? c : cap;
        k_max = K[i] > k_max ? K[i] : k_max;
    }
    std::vector<Block> full((size_t)cap);
    return pool_table_cap(aligned, bounds ? b.data() : nullptr, N, P, K, n, win_len, k_max, full.data());
}

// A banked source (spectra of K = ceil(L / 4096) partitions per row) rendered into out (C, win_len) as a pooled slot of a
// pool with mixed K renders it: grid blocking, the window's blocks of its own K, and k_render<LONG> (long = 1) or the
// kernel it would run alone (long = 0).
int emu_render_slot(const float* x, const float2* spec, float* out, const int32_t* bounds, int N, int P, int C, int L,
                    int mode, int win_start, int win_len, int long_variant) {
    const Tables& T = tables();
    Source S;
    memset(&S, 0, sizeof(S));
    S.x = x; S.out = out; S.bounds = bounds;
    S.N = N; S.P = P; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.nb = (N + kB - 1) / kB; S.mode = mode;
    const int cap = table_cap(0, S.nb, P);
    std::vector<Block> full((size_t)cap);
    const int nfull = plan_blocks(0, bounds, P, N, S.nb, 0, cap, full.data());
    const WinSpan ws = window_blocks(full.data(), nfull, win_start, win_start + win_len, S.K);
    S.nblk_max = ws.g1 - ws.g0;
    std::vector<Block> blocks((size_t)S.nblk_max);
    const int nplan = plan_blocks(0, bounds, P, N, S.nb, ws.g0, ws.g1, blocks.data());
    const int nblk = (nplan < ws.g1 ? nplan : ws.g1) - ws.g0;
    clear_blocks(blocks.data(), nblk, S.nblk_max, 0, 1);
    std::vector<double> rstep((size_t)P);
    if (mode == MODE_MOVING_BOUNDS) fill_rstep(bounds, P, rstep.data(), 0, 1);
    int counts[16] = {nblk, 0, ws.k0 - ws.g0, ws.k1 - ws.k0, win_start, win_len};
    const float one = 1.0f;
    memcpy(counts + 11, &one, sizeof(one));
    S.blocks = blocks.data(); S.rstep = rstep.data(); S.counts = counts;
    set_banked(S, const_cast<float2*>(spec), nullptr, true);
    std::vector<float2> xs((size_t)S.nblk_max * kSpec);
    S.xspec = xs.data();
    std::vector<RItem> items((size_t)max_render_items(S));
    for (int i = 0; i < spectra_pairs_x(S); ++i) cta_spectra(S, i, T);
    prepare_ranges(S, items.data());
    const int nr = win_blocks(S) * items_per_block(S);
    const int grid = nr < 3 ? nr : 3;
    for (int cta = 0; cta < grid; ++cta) {
        if (!long_variant && one_transform_per_item(0, mode, S.K)) cta_render_fast(items.data(), nr, cta, grid, T);
        else cta_render(items.data(), nr, cta, grid, T, false, long_variant || S.K > 1);
    }
    return 0;
}

}  // extern "C"
