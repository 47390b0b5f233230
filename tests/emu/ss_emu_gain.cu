// tests/emu/ss_emu_gain.cu - the loudness gain of a pooled slot (ss_pool_loudness) in the emulated kernels.
//
// TEST INFRASTRUCTURE, like ss_emu.cu, whose emulated source driver it runs (through ss_emu_window.cu, included below)
// with one change: the emulated k_prepare hands fill_items the gain set by emu_set_gain, as the kernel hands it
// stem_gain(S), so that every work item - and every epilogue branch that stores from it - carries that gain.  Also
// exports the head of k_blocks for a pooled slot (pick_slot).  Built with g++ (`-x c++`) by tests/test_pool_loudness.py.
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

static float g_emu_gain = 1.0f;
// every call of fill_items below (k_prepare's range warps in ss_emu.cu) passes the gain; the name is not re-expanded
#define fill_items(...) fill_items(__VA_ARGS__, g_emu_gain)

#include "ss_emu_window.cu"

#undef fill_items

extern "C" {

void emu_set_gain(float g) { g_emu_gain = g; }

// pick_slot on a slot over a pool of n candidates (candidate i has N = 1000 + i) whose gains are `gains` (null: a pool
// without gains): out[0] = the picked candidate's index (from N), out[1] = 1 if the pick was clamped, and *gain_out the
// gain the slot's counts then hold (stem_gain)
int emu_pick_slot(int v, int n, const float* gains, int* out, float* gain_out) {
    std::vector<PoolEntry> pool((size_t)n);
    static float x[1];
    static float2 spec[1];
    for (int i = 0; i < n; ++i) {
        pool[i].x = x; pool[i].bounds = nullptr; pool[i].spec = spec; pool[i].cut = nullptr;
        pool[i].N = 1000 + i; pool[i].P = 1;
    }
    int counts[16] = {};
    const PoolEntry* table = pool.data();
    memcpy(counts + 8, &table, sizeof(table));
    counts[10] = n;
    const int* pick = &v;
    memcpy(counts + 12, &pick, sizeof(pick));
    memcpy(counts + 14, &gains, sizeof(gains));
    Source s;
    memset(&s, 0, sizeof(s));
    s.C = 1; s.K = 1; s.counts = counts;
    bool bad = false;
    pick_slot(s, *pick_ptr(s), bad);
    out[0] = s.N - 1000; out[1] = bad ? 1 : 0;
    *gain_out = stem_gain(s);                     // s.h_rows is set: a pooled slot is a windowed source
    return 0;
}

}  // extern "C"
