// tests/emu/ss_emu_traj.cu - trajectories of pooled slots (ss_trajectory) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE, like ss_emu_bank.cu, whose bank builder and emulated phases it reuses (included below).  Exports
// the table-size rule of a slot with a trajectory (traj_table_cap) and a pooled slot of a one-candidate pool rendered as
// the plan renders it: the head of k_blocks (pick_pooled, then take_trajectory), the window's blocks of the full plan
// over the slot's bounds after the head, k_prepare's dry-window CTAs, the slot's items (fill_traj_items, as k_blocks
// fills them; k_prepare's range warps then skip the slot) and the render CTAs.
// Built with g++ (`-x c++`) by tests/test_trajectory.py.
#include "ss_emu_bank.cu"

extern "C" {

// traj_table_cap over n candidates (N[i], P[i], K[i] partitions) with windows of win_len
int emu_traj_table_cap(const int* N, const int* P, const int* K, int n, int aligned, int win_len) {
    int cap = 0, k_max = 0;
    for (int i = 0; i < n; ++i) {
        const int c = table_cap(aligned, (N[i] + kB - 1) / kB, P[i]);
        cap = c > cap ? c : cap;
        k_max = K[i] > k_max ? K[i] : k_max;
    }
    std::vector<Block> full((size_t)cap);
    return traj_table_cap(aligned, N, P, K, n, win_len, k_max, full.data());
}

// A slot of C channels over a pool holding one banked candidate (dry x of N samples, P positions, bounds, spectra
// `spec` of K = ceil(L / 4096) partitions), window [ws, ws + wl), under aligned (K == 1) or grid blocking.  path null:
// no trajectory; else path (a, b, dir) and tbounds as the slot's device arrays.  out receives (C, wl); info receives
// [error bits of the head, blocks the window's table needs, the slot's P after the head, reverse flag].
int emu_traj_render(const float* x, const float2* spec, float* out, const int32_t* bounds, const int32_t* path,
                    const int32_t* tbounds, int N, int P, int C, int L, int aligned, int ws, int wl, int* info) {
    const Tables& T = tables();
    PoolEntry e;
    e.x = x; e.bounds = bounds; e.spec = const_cast<float2*>(spec); e.cut = nullptr; e.N = N; e.P = P;
    int counts[32] = {};
    const PoolEntry* table = &e;
    memcpy(counts + 8, &table, sizeof(table));
    counts[10] = 1;
    const int v = 0;
    const int* pick = &v;
    memcpy(counts + 12, &pick, sizeof(pick));
    counts[4] = ws; counts[5] = wl;
    if (path) {
        counts[25] = 1;
        memcpy(counts + 28, &path, sizeof(path));
        memcpy(counts + 30, &tbounds, sizeof(tbounds));
    }
    Source S;
    memset(&S, 0, sizeof(S));
    S.out = out; S.C = C; S.L = L; S.K = (L + kB - 1) / kB; S.mode = MODE_MOVING_BOUNDS; S.aligned = aligned;
    S.counts = counts;
    S.h_rows = 1;                                         // a windowed source until the pick sets its rows
    unsigned err = pick_pooled(S);
    if (has_traj(S)) err |= take_trajectory(S);
    // the window's blocks of the full plan over the slot's bounds, as k_blocks writes them
    const int cap = table_cap(aligned, S.nb, S.P);
    std::vector<Block> full((size_t)cap);
    const int nfull = plan_blocks(aligned, S.bounds, S.P, S.N, S.nb, 0, cap, full.data());
    const WinSpan w = window_blocks(full.data(), nfull, ws, ws + wl, S.K);
    S.nblk_max = w.g1 - w.g0;
    std::vector<Block> blocks((size_t)S.nblk_max);
    for (int i = w.g0; i < w.g1; ++i) blocks[i - w.g0] = full[i];
    std::vector<double> rstep((size_t)S.P);
    fill_rstep(S.bounds, S.P, rstep.data(), 0, 1);
    counts[0] = S.nblk_max; counts[1] = 0; counts[2] = w.k0 - w.g0; counts[3] = w.k1 - w.k0;
    S.blocks = blocks.data(); S.rstep = rstep.data();
    std::vector<float2> xs((size_t)S.nblk_max * kSpec);
    S.xspec = xs.data();
    std::vector<RItem> items((size_t)max_render_items(S));
    for (int i = 0; i < spectra_pairs_x(S); ++i) cta_spectra(S, i, T);
    if (has_traj(S)) {                                    // k_blocks fills the items, k_prepare's range warps skip them
        fill_traj_items(S, items.data(), 0, 1);
        counts[0] = 0;
    }
    prepare_ranges(S, items.data());
    const int nr = win_blocks(S) * items_per_block(S);
    const int grid = nr < 3 ? nr : 3;
    for (int cta = 0; cta < grid; ++cta) {
        if (one_transform_per_item(aligned, S.mode, S.K)) cta_render_fast(items.data(), nr, cta, grid, T);
        else cta_render(items.data(), nr, cta, grid, T, false, S.K > 1);
    }
    info[0] = (int)err; info[1] = S.nblk_max; info[2] = S.P; info[3] = (counts[25] & 2) ? 1 : 0;
    return 0;
}

}  // extern "C"
