// tests/emu/ss_emu_moving.cu - the planning helpers of a moving window (ss_source.win_start_dev) on the CPU.
//
// TEST INFRASTRUCTURE: exports the functions of ss_phases.cuh that size a moving window's block table
// (window_table_cap, over the full plan of plan_blocks), find the table a given start needs (window_blocks, as the
// host planner and k_blocks find it) and clamp a start read from device memory (clamp_win_start, as k_blocks does).
// Built with g++ (`-x c++`) by tests/test_moving_window.py.
#include <math.h>
#include <stdint.h>
#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

// the full plan of a source (aligned: from its bounds) into `full`; returns its block count
static int full_plan(const int32_t* bounds, int N, int P, int aligned, std::vector<Block>& full) {
    const int nb = (N + kB - 1) / kB;
    full.resize((size_t)table_cap(aligned, nb, P));
    const int n = plan_blocks(aligned, bounds, P, N, nb, 0, (int)full.size(), full.data());
    return n < (int)full.size() ? n : (int)full.size();
}

extern "C" {

// Table size the library gives a moving window of win_len samples.  host_plan: the full plan is known on the host
// (grid blocking, or aligned blocking with bounds_host); otherwise the device bound of aligned blocking.
int emu_window_table_cap(const int32_t* bounds, int N, int P, int L, int aligned, int host_plan, int win_len) {
    const int K = (L + kB - 1) / kB, nb = (N + kB - 1) / kB;
    std::vector<Block> full;
    const int n = host_plan ? full_plan(bounds, N, P, aligned, full) : 0;
    return window_table_cap(host_plan ? full.data() : nullptr, n, N, win_len, K, P, table_cap(aligned, nb, P));
}

// g1 - g0 of window_blocks for every start in [0, N - win_len] into need[] (N - win_len + 1 entries): the table each
// start's blocks take
int emu_window_tables(const int32_t* bounds, int N, int P, int L, int aligned, int win_len, int* need) {
    std::vector<Block> full;
    const int n = full_plan(bounds, N, P, aligned, full);
    for (int ws = 0; ws <= N - win_len; ++ws) {
        const WinSpan w = window_blocks(full.data(), n, ws, ws + win_len, (L + kB - 1) / kB);
        need[ws] = w.g1 - w.g0;
    }
    return 0;
}

// k_blocks' clamp of a start read from device memory; *bad = 1 when it was outside [0, N - win_len]
int emu_clamp_win_start(int v, int N, int win_len, int* bad) {
    bool b = false;
    const int r = clamp_win_start(v, N, win_len, b);
    *bad = b ? 1 : 0;
    return r;
}

}  // extern "C"
