// tests/emu/ss_emu_values.cu - value draws of plans (ss_value_draw) in the emulated kernels, on the CPU.
//
// TEST INFRASTRUCTURE: runs what k_values runs - value_row of ss_phases.cuh over every row and draw, in list order,
// with the plan's descriptors filled as plan_build fills them.  Built with g++ (`-x c++`) by tests/value_reference.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "../../include/sonicsim_b200.h"
#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// Every row of the n value draws `values` (host out, base and rng_dev pointers), as k_values writes them: row by row,
// draw after draw, each row's elements split over `lanes` lanes that run one after the other.
void emu_value_rows(const ss_value_draw* values, int n, int lanes) {
    std::vector<ValueDesc> descs(n);
    for (int k = 0; k < n; ++k) {                        // (as plan_build fills them)
        const ss_value_draw& v = values[k];
        ValueDesc& g = descs[k];
        memset(&g, 0, sizeof(g));
        g.out = v.out; g.rng = v.rng_dev;
        g.base = v.base >= 0 ? (const int*)values[v.base].out : nullptr;
        g.low = v.low; g.high = v.high; g.ilow = v.ilow; g.n = (uint32_t)((int64_t)v.ihigh - v.ilow);
        g.kind = v.kind; g.k = v.k; g.r = k; g.stride = v.base >= 0 ? v.stride : 0;
    }
    uint32_t map[2 * kValueMapCap];
    for (int b = 0; b < (n ? values[0].rows : 0); ++b)
        for (int k = 0; k < n; ++k)
            for (int lane = 0; lane < lanes; ++lane) value_row(descs[k], b, lane, lanes, map, map + kValueMapCap);
}

// The word of element j of row b of value draw r at (seed, t)
uint64_t emu_value_word(int64_t seed, int64_t t, int r, int b, int j) {
    return value_word((uint32_t)(uint64_t)seed, (uint32_t)((uint64_t)seed >> 32), (uint32_t)(uint64_t)t,
                      (uint32_t)((uint64_t)t >> 32), r, b, j);
}

// The values of word x: float64, float32, and the integer in [0, n)
double emu_value_f64(double low, double high, uint64_t x) { return value_f64(low, high, x); }
float emu_value_f32(double low, double high, uint64_t x) { return value_f32(low, high, x); }
uint64_t emu_value_below(uint64_t x, uint64_t n) { return umulhi64(x, n); }

}  // extern "C"
