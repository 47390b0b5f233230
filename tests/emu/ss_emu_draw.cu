// tests/emu/ss_emu_draw.cu - the start draw of a device plan (ss_plan_draw) on the CPU.
//
// TEST INFRASTRUCTURE: runs the per-try functions of ss_phases.cuh that k_draw runs in its lanes (draw_span, draw_start,
// draw_silent) one try after the other, as the dataloader's loop does (movingdatamodule.py:81-99).  Built with g++
// (`-x c++`) by tests/test_plan_draw.py.
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "../../sonicsim_b200/csrc/ss_phases.cuh"

using namespace ss;

extern "C" {

// One draw: S speakers with level tables Q[k] and crop element counts D[k]; the picked N of each of n_readers readers;
// tries uniform variates u.  Returns the start, *used the 1-based index of the kept try or 0.
int emu_draw(const double* const* Q, const double* D, int S, const int* reader_N, int n_readers, int len,
             const double* u, int tries, float threshold_db, int* used) {
    int M = 0x7fffffff;
    for (int r = 0; r < n_readers; ++r) { const int m = draw_span(reader_N[r], len); M = m < M ? m : M; }
    int s = 0;
    for (int t = 0; t < tries; ++t) {
        s = draw_start(u[t], M);
        bool silent = false;
        for (int k = 0; k < S; ++k) silent = silent || draw_silent(Q[k], s, len, D[k], threshold_db);
        if (!silent) { *used = t + 1; return s; }
    }
    *used = 0;
    return s;
}

int emu_draw_start(double u, int M) { return draw_start(u, M); }

}  // extern "C"
