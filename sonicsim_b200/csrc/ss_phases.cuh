// sonicsim_b200 :: ss_phases.cuh
//
// The kernels of the renderer, cut into barrier-free *phases*.  A phase is a function of one
// thread id, that thread's registers (a struct) and the CTA's shared array.  ss_kernels.cu calls
// the phases with __syncthreads() between them; tests/emu/ss_emu.cu calls the same phases in a
// `for (tid)` loop per phase.  All addressing and arithmetic is therefore tested on the CPU.
#pragma once
#include "ss_core.cuh"

namespace ss {

enum { MODE_STATIC = 0, MODE_MOVING_BOUNDS = 1, MODE_MOVING_INDEXED = 2 };

// One output block: samples [start, start + len), len <= 4096, rendered by one transform per pair of
// positions in [p_lo, p_hi].  len == 0: unused slot of the table.
//   grid blocking     start = 4096 b                     (long RIRs, indexed trajectories, static sources)
//   aligned blocking  blocks never cross a waypoint: every block lies in one segment s and needs
//                     exactly the pair (s, s + 1) -> one transform, both packed results used
//                     (bounds trajectory and L <= 4096)
struct Block { int start, len, p_lo, p_hi; };

struct RItem;

// One (utterance, source) unit.  Reference shapes: dry (N,), RIRs (P, C, L), output (C, N)
// (SonicSim_moving.py:63-96); static source has P = 1 (SonicSim_moving.py:47-61).
// Biased pointers: the kernels index x, rir, idx and w as the full arrays (sample n at x[n], position p at
// rir + p * C * L), but for a windowed source the host path copies only its read set, so these four may point in
// front of their allocation (device buffer - first index copied), and RItem::row / row1 point win_start samples in
// front of the (C, win_len) output.  Only indices inside the read set / the window are ever dereferenced; code that
// reads any other element of these arrays must first be added to the read set (include/sonicsim_b200.h).
struct Source {
    const float* x;        // dry waveform, N samples
    const float* rir;      // (P, C, L) row-major
    float* out;            // (C, N) row-major, channel-major like torchaudio.save expects
    const int* bounds;     // compact trajectory: S+1 cumulative segment bounds (mode 1), else null
    const int* idx;        // per-sample interp_index  (mode 2), else null
    const float* w;        // per-sample interp_weight (mode 2), else null
    float2* hspec;         // scratch: P*C*K half spectra of the RIR partitions, pre-scaled by 1/F; a direct-target
                           // source has a second P*C*K block right behind it for the direct rows (same layout)
    float2* xspec;         // scratch: nblk_max half spectra of the dry windows
    Block* blocks;         // scratch: nblk_max blocks (k_blocks)
    double* rstep;         // scratch: 1 / (samples in segment s), s < P - 1 (mode 1)
    int* counts;           // scratch: [0] = blocks in use, [1] = index of this source's first render item; windowed
                           // source (h_rows != 0): [2] = first block that meets the window, [3] = blocks that do,
                           // [4] = win_start, [5] = win_len, [6..7] = device pointer of a moving window's start or
                           // null (win_start_ptr); tables built on the device: [8..17] the pool of a pooled slot
                           // (pool_table, pool_size, pick_ptr, pool_gains, pool_parts), [18..19] its stage view,
                           // [20..24] its dry pick (dry_table, dry_pick_ptr, dry_size)
    const float* norm_part;// scratch: kNormParts partial abs-maxima of the RIR tensor (k_rir_absmax), or null: taps used as given
    int* cut;              // scratch: P*C direct-path row lengths (k_rir_direct), or null: no direct target
    float* out_direct;     // (C, N) direct-path stem (with `cut`)
    int N, P, C, L;
    int K;                 // RIR partitions = ceil(L / kB)
    int nb;                // ceil(N / kB)
    int mode;              // 0 static, 1 moving (bounds), 2 moving (idx, w)
    int aligned;           // 1: blocks aligned to the trajectory segments (mode 1 and K == 1)
    int nblk_max;          // table size: nb (grid) or nb + P - 1 (aligned)
    int direct_taps;       // taps kept from each row's peak on (with `cut`)
    // Time window (0, 0: the whole stem).  A windowed source transforms only the RIR rows [h_row0, h_row0 + h_rows) of
    // each set (h_row0 even: rows pair as in the full row list), stored from hspec on, and only a contiguous range of
    // the full plan's blocks (k_blocks / the host: first block even, see window_span); out / out_direct are
    // (C, win_len).  h_rows != 0 marks a windowed source.
    int h_row0, h_rows;
};
// A banked source (ss_bank, include/sonicsim_b200.h) has rir == null: hspec (and cut, with a direct target) point into
// the bank, which holds all P*C*K rows of each set from row 0 - what a whole source transforms into its scratch - so
// k_prepare transforms none of its rows (spectra_pairs_h == 0), k_rir_direct skips it and it has no norm_part.  Windowed
// or not, the set stride and row origin are the bank's: h_row0 = 0, and h_rows = P*C*K when windowed (still nonzero,
// it marks the window).  Needs P, C and K set.
SS_HD void set_banked(Source& s, float2* spec, int* cut, bool windowed) {
    s.rir = nullptr; s.hspec = spec; s.cut = cut; s.norm_part = nullptr;
    s.h_row0 = 0; s.h_rows = windowed ? s.P * s.C * s.K : 0;
}
constexpr int kNormParts = 128;    // CTAs (partial maxima) per normalised source in k_rir_absmax

// One unit of k_render work: one block of channel c (static: channels c, c+1), written by k_prepare
// so that k_render never searches trajectories, prefix tables or the Source array.
struct RItem {
    const float2* X;       // dry spectrum of the block's window [start - 4096, start + 4096)
    const float2* H0;      // RIR spectrum of (position 0, channel c, partition 0); position p at H0 + p * pstride
    float* row;            // output row of channel c
    float* row1;           // static source: output row of channel c + 1, or null
    const int* bounds;     // trajectory of the source (mode 1)
    const double* rstep;   //   "
    const int* idx;        // (mode 2)
    const float* w;        // (mode 2)
    int pstride;           // float2 words between positions (moving: C*K*kSpec, negated for a reverse trajectory:
                           // fill_traj_items) / to channel c+1 (static: K*kSpec); applied as a signed product
    int n0, n_end;         // output samples [n0, n_end)
    int p_lo, p_hi;        // transforms p = p_lo, p_lo + 2, ... <= p_hi   (static: 0, 0)
    int mode;
    int kparts;            // RIR partitions that reach back into the signal: min(K, n0 / 4096 + 1)
    int b0;                // aligned blocking: first sample of the block's segment, bounds[p_lo] ...
    double step;           // ... and 1 / (samples in that segment), so that k_render_fast's output stage loads no table
    int n_lo;              // samples [n_lo, n_end) are stored (n_lo > n0: a window starts inside the block); the
                           // epilogues tie register r to sample n0 + t + 256 r, so n0 stays the block start
    float gain;            // every stored sample is scaled by it (gain_mul): a pooled slot's loudness gain, else 1
};
static_assert(sizeof(RItem) == 112, "RItem is copied as 7 x 16 B");

// One inverse transform, published by the CTA's thread 0 to the other threads through shared memory.
struct XDesc {
    const float2* X;       // global pointers, used for RIR partitions >= 1 (partition 0 is staged by TMA)
    const float2* Hp;
    const float2* Hq;      // null: only one filter packed into this transform
    float* row;
    float* row1;
    const int* bounds;
    const double* rstep;
    const int* idx;
    const float* w;
    int n0, n_end, p, p_lo, p_hi;
    int first;             // first transform of its block: plain store, otherwise accumulate
    int valid;
    int mode;
    int kparts;
    int n_lo;              // as RItem::n_lo
    float gain;            // as RItem::gain
    int pad_;
};
static_assert(sizeof(XDesc) == 120, "XDesc layout");

// RIR rows are transformed two per complex FFT, and the bits of a half spectrum depend on its partner row: the direct
// rows are paired among themselves exactly as a separate source's rows would be, never with a reverberant row.
SS_HD int rows_h(const Source& s) { return s.P * s.C * s.K; }                 // per set (reverberant, direct)
SS_HD int rows_stored_h(const Source& s) { return s.h_rows ? s.h_rows : rows_h(s); }     // transformed rows per set
SS_HD int pairs_per_set_h(const Source& s) { return (rows_stored_h(s) + 1) >> 1; }
SS_HD int spectra_pairs_h(const Source& s) { return s.rir ? pairs_per_set_h(s) * (s.cut ? 2 : 1) : 0; }   // banked: 0
SS_HD int spectra_pairs_x(const Source& s) { return (s.nblk_max + 1) >> 1; }
SS_HD int range_ctas(const Source& s) { return (s.nblk_max + 7) >> 3; }       // k_prepare: one warp per block
SS_HD int items_per_set(const Source& s) { return s.mode == MODE_STATIC ? (s.C + 1) >> 1 : s.C; }
SS_HD int items_per_block(const Source& s) { return items_per_set(s) * (s.cut ? 2 : 1); }
SS_HD int max_render_items(const Source& s) { return s.nblk_max * items_per_block(s); }
// Every render item of the source needs one inverse transform (k_render_fast): aligned blocking, or a static source
// with one RIR partition.  Everything else goes through k_render, with LONG when K > 1.
SS_HD bool one_transform_per_item(int aligned, int mode, int K) { return aligned || (mode == MODE_STATIC && K == 1); }

// ---- the block table: one planner for the host, k_blocks and the CPU emulation.
// blocks of one segment under aligned blocking
SS_HD int seg_blocks(int n_s) { return (n_s + kB - 1) / kB; }
// block q of segment sg = [b0, b0 + n_s) under aligned blocking
SS_HD Block seg_block(int b0, int n_s, int q, int sg) {
    Block bk; bk.start = b0 + kB * q; bk.len = n_s - kB * q < kB ? n_s - kB * q : kB; bk.p_lo = sg; bk.p_hi = sg + 1;
    return bk;
}
// block bi of an N-sample source under grid blocking (its positions are found by k_prepare's range warps)
SS_HD Block grid_block(int N, int bi) {
    Block bk; bk.start = bi * kB; bk.len = N - bi * kB < kB ? N - bi * kB : kB; bk.p_lo = 0; bk.p_hi = 0;
    return bk;
}
// table size of a whole source: nb (grid), nb + P - 1 (aligned: at most one partial block per waypoint)
SS_HD int table_cap(int aligned, int nb, int P) { return aligned ? nb + P - 1 : nb; }
// unused slots [n, cap) of a table (lane `lane` of `nlanes`)
SS_HD void clear_blocks(Block* b, int n, int cap, int lane, int nlanes) {
    for (int bi = n + lane; bi < cap; bi += nlanes) { Block z; z.start = 0; z.len = 0; z.p_lo = 0; z.p_hi = 0; b[bi] = z; }
}
// 1 / (samples in segment sg) for every segment of a bounds trajectory (lane `lane` of `nlanes`)
SS_HD void fill_rstep(const int* bounds, int P, double* rstep, int lane, int nlanes) {
    for (int sg = lane; sg < P - 1; sg += nlanes) rstep[sg] = 1.0 / (double)(bounds[sg + 1] - bounds[sg]);
}
// The full plan's blocks with index in [g0, g1), written to out[0 ..]; returns the full plan's block count (whole
// source: g0 = 0, g1 = table_cap).  Aligned blocking reads the bounds, grid blocking does not.
SS_HD int plan_blocks(int aligned, const int* bounds, int P, int N, int nb, int g0, int g1, Block* out) {
    if (!aligned) {
        for (int bi = g0; bi < g1 && bi < nb; ++bi) out[bi - g0] = grid_block(N, bi);
        return nb;
    }
    int n = 0;
    for (int sg = 0; sg < P - 1; ++sg) {
        const int b0 = bounds[sg], n_s = bounds[sg + 1] - b0;
        for (int q = 0; q < seg_blocks(n_s); ++q, ++n)
            if (n >= g0 && n < g1) out[n - g0] = seg_block(b0, n_s, q, sg);
    }
    return n;
}

// ---- time windows.  A windowed source keeps the full plan's blocking (aligned or grid, chosen over the whole
// trajectory) and renders the blocks [k0, k1) of the full table that meet the window.  Its table holds the full
// table's blocks [g0, g1): the K - 1 blocks in front of k0 too (their dry windows feed RIR partitions 1 .. K - 1), g0
// even and g1 past the last kept block's partner, because two dry windows share one forward FFT - blocks 2i and 2i + 1
// of the full table - and the bits of each half spectrum depend on its partner.
struct WinSpan { int g0, g1, k0, k1; };
SS_HD WinSpan window_span(int k0, int k1, int nblk, int K) {
    WinSpan r; r.k0 = k0; r.k1 = k1;
    const int a = k0 - (K - 1);
    r.g0 = (a > 0 ? a : 0) & ~1;
    r.g1 = (k1 + 1) & ~1;
    if (r.g1 > nblk) r.g1 = nblk;
    return r;
}
// the same from the full table itself (ascending starts, no empty block): the blocks meeting output samples [ws, we)
SS_HD WinSpan window_blocks(const Block* b, int nblk, int ws, int we, int K) {
    int lo = 0, hi = nblk;                               // first block that ends after ws
    while (lo < hi) { const int m = (lo + hi) >> 1; if (b[m].start + b[m].len <= ws) lo = m + 1; else hi = m; }
    const int k0 = lo;
    hi = nblk;                                           // first block that starts at or after we
    while (lo < hi) { const int m = (lo + hi) >> 1; if (b[m].start < we) lo = m + 1; else hi = m; }
    return window_span(k0, lo, nblk, K);
}
// first RIR row and row count of a windowed source whose kept blocks interpolate between positions [pa, pb]: whole
// positions, started on an even row and ended past the last row's partner (rows 2r, 2r + 1 share one forward FFT)
SS_HD void window_rows(int P, int C, int K, int pa, int pb, int& row0, int& rows) {
    const int ck = C * K;
    const int r0 = (pa * ck) & ~1;
    int r1 = ((pb + 1) * ck + 1) & ~1;
    if (r1 > P * ck) r1 = P * ck;
    row0 = r0; rows = r1 - r0;
}
// Table size that holds the window's blocks [g0, g1) whatever its start in [0, N - win_len] (a moving window: the start
// is read on the device at every run, the table is sized once).  full / nfull: the full plan's blocks when the host
// knows them (grid blocking, or aligned blocking with bounds_host) - they tile [0, N), and for a fixed first block k0
// g1 - g0 grows with the start, so one sliding pass over the largest start of each k0 gives the exact maximum.  Under
// grid blocking that is at most ceil(win_len / 4096) + K + 2 (one straddling block, K - 1 partition blocks and the
// even rounding in front, the partner behind).  full == null (aligned blocking over device-side bounds): a window
// meets at most ceil(o / 4096) + 1 blocks of each segment it overlaps by o samples, plus one block in front (even
// start) and the last one's partner.  Never more than `cap`, the whole source's table.
SS_HD int window_table_cap(const Block* full, int nfull, int N, int win_len, int K, int P, int cap) {
    if (!full) {
        const int64_t bound = (int64_t)(win_len + kB - 1) / kB + 2 * (int64_t)(P - 1) + 2;
        return bound < cap ? (int)bound : cap;
    }
    int best = 0, k1 = 0;
    for (int k0 = 0; k0 < nfull && full[k0].start <= N - win_len; ++k0) {
        const int end = full[k0].start + full[k0].len - 1;
        const int we = (end < N - win_len ? end : N - win_len) + win_len;   // largest start whose first block is k0
        while (k1 < nfull && full[k1].start < we) ++k1;
        const WinSpan w = window_span(k0, k1, nfull, K);
        best = w.g1 - w.g0 > best ? w.g1 - w.g0 : best;
    }
    return best < cap ? best : cap;
}
// A moving window's start as read from device memory, clamped into [0, N - win_len]; bad = it was outside
SS_HD int clamp_win_start(int v, int N, int win_len, bool& bad) {
    const int hi = N - win_len;
    bad = v < 0 || v > hi;
    return v < 0 ? 0 : (v > hi ? hi : v);
}
// a windowed source's moving start (counts[6..7], 8-byte aligned), or null: the start is counts[4]
SS_HD const int* win_start_ptr(const Source& s) { return *reinterpret_cast<const int* const*>(s.counts + 6); }

// ---- loudness slots of plans (ss_stream_lufs): a stream or bed slot is rendered whole, [0, N), into plan scratch,
// measured there at every run (k_kweight, k_kw_scan, k_loud_gate<true>), and k_loud_crop cuts its crop out of the
// whole stem with the gain of that run.  One descriptor per slot:
struct LoudCrop {
    const float* whole;        // (C, N) the slot's whole stem ...
    const float* whole_dir;    // ... and its whole direct-path stem, or null
    float* out;                // (C, len) the slot's crop ...
    float* out_dir;            // ... and its direct-path crop, or null
    const int* ws_dev;         // the slot's moving start, or null: ws
    const double* target;      // the target LUFS, read at every run
    const double* result;      // (LUFS, gain) that k_loud_gate<true> wrote at this run
    int ws, len, N, C;
};
// Head of k_loud_crop: the crop's start, clamped as a pooled window's start is (bit 2), and the float32 gain of the
// crops, (float)result[1] as k_loud_scale takes it, or 1 with bit 6 for a non-finite target (stored unscaled).
// Returns the error bits.
SS_HD unsigned loud_crop_head(const LoudCrop& q, int& start, float& g) {
    unsigned err = 0;
    start = q.ws;
    if (q.ws_dev) {
        bool bad;
        start = clamp_win_start(*q.ws_dev, q.N, q.len, bad);
        if (bad) err |= 4u;
    }
    const double t = *q.target;
    if (isfinite(t)) g = (float)q.result[1];
    else { g = 1.0f; err |= 64u; }
    return err;
}
// element i of set `dir` (0: the stem, 1: the direct-path stem) of a crop: channel i / len, sample i % len
SS_HD float loud_crop_sample(const LoudCrop& q, int start, float g, int dir, long long i) {
    const long long c = i / q.len, t = i - c * q.len;
    return (dir ? q.whole_dir : q.whole)[c * q.N + start + t] * g;
}

// ---- source pools (ss_pool, include/sonicsim_b200.h).  A pooled slot is a windowed source whose candidate is picked on
// the device at every run: the head of k_blocks reads the pick, clamps it and writes the candidate's fields into the
// slot's Source (pick_candidate) before anything reads them.  One compact entry per candidate in the pool's table:
struct PoolEntry {
    const float* x;        // dry signal, N samples
    const int* bounds;     // trajectory bounds (moving pool), else null
    float2* spec;          // the bank's spectra (reverberant set, then the direct set)
    int* cut;              // the bank's direct-path cut table, or null: no direct set
    int N, P;
};
static_assert(sizeof(PoolEntry) == 40, "PoolEntry layout");
// A pooled slot's counts (counts_bytes = 64 for every windowed source whose tables k_blocks builds, 80 for a pooled slot):
// [8..9] the pool's device table or null (not pooled), [10] its candidate count, [12..13] the device pointer of the pick
SS_HD const PoolEntry* pool_table(const Source& s) { return *reinterpret_cast<const PoolEntry* const*>(s.counts + 8); }
SS_HD int pool_size(const Source& s) { return s.counts[10]; }
SS_HD const int* pick_ptr(const Source& s) { return *reinterpret_cast<const int* const*>(s.counts + 12); }
// A pick as read from device memory, clamped into [0, n); bad = it was outside
SS_HD int clamp_pick(int v, int n, bool& bad) {
    bad = v < 0 || v >= n;
    return v < 0 ? 0 : (v >= n ? n - 1 : v);
}
// The picked candidate into the slot's Source, as set_banked sets a windowed banked source (K, C, mode, aligned and the
// slot's own buffers stay): the direct set only for a slot that renders a direct stem
SS_HD void pick_candidate(Source& s, const PoolEntry& e) {
    s.x = e.x; s.bounds = e.bounds; s.N = e.N; s.P = e.P; s.nb = (e.N + kB - 1) / kB;
    set_banked(s, e.spec, s.out_direct ? e.cut : nullptr, true);
}
// Loudness gains (ss_pool_loudness): a windowed source's counts[11] holds the float bits of the gain its stems are
// stored with - 1 (written by the host) unless a pooled slot picked a candidate of a pool with gains - and a pooled slot's
// [14..15] the device pointer of its pool's n float gains, or null
SS_HD const float* pool_gains(const Source& s) { return *reinterpret_cast<const float* const*>(s.counts + 14); }
SS_HD float stem_gain(const Source& s) { return s.h_rows ? *reinterpret_cast<const float*>(s.counts + 11) : 1.0f; }
SS_HD void set_stem_gain(Source& s, float g) { *reinterpret_cast<float*>(s.counts + 11) = g; }
// The head of k_blocks for a pooled slot: the pick v read from device memory, clamped into [0, n) (bad = it was not
// there), the picked candidate written into the slot's Source and its gain into counts[11] (1 for a pool without gains)
SS_HD void pick_slot(Source& s, int v, bool& bad) {
    const int i = clamp_pick(v, pool_size(s), bad);
    pick_candidate(s, pool_table(s)[i]);
    const float* const g = pool_gains(s);
    set_stem_gain(s, g ? g[i] : 1.0f);
}
// Candidates of one pool may differ in L.  A pool whose candidates differ in K (RIR partitions) keeps a device array of
// their n partition counts; a pooled slot's counts block is 80 bytes, and [16..17] hold that array's device pointer, or
// null (a uniform pool: the slot keeps the pool's K).  The head of k_blocks sets the slot's K to the picked candidate's
// (pick_parts) before pick_slot, whose set_banked derives h_rows = P*C*K from it; the window search, the block table and
// fill_items (kparts, pstride, the direct set's offset) then follow the picked K.
SS_HD const int* pool_parts(const Source& s) { return *reinterpret_cast<const int* const*>(s.counts + 16); }
SS_HD void pick_parts(Source& s, int v) {
    const int* const k = pool_parts(s);
    bool bad;
    if (k) s.K = k[clamp_pick(v, pool_size(s), bad)];
}
// Table size of a pooled slot with windows of win_len: the largest window_table_cap over the candidates' full plans under
// the pool's blocking (bounds[i]: candidate i's host bounds, null for a static pool), so that the table holds the blocks
// of every candidate at every start.  Candidate i has Ks[i] RIR partitions (g1 - g0 grows with K), or K when Ks is null.
// `full` holds table_cap(aligned, nb, P) blocks of the largest candidate.
SS_HD int pool_table_cap(int aligned, const int* const* bounds, const int* N, const int* P, const int* Ks, int n,
                         int win_len, int K, Block* full) {
    int best = 0;
    for (int i = 0; i < n; ++i) {
        const int nb = (N[i] + kB - 1) / kB, cap = table_cap(aligned, nb, P[i]);
        const int nfull = plan_blocks(aligned, bounds ? bounds[i] : nullptr, P[i], N[i], nb, 0, cap, full);
        const int c = window_table_cap(full, nfull < cap ? nfull : cap, N[i], win_len, Ks ? Ks[i] : K, P[i], cap);
        best = c > best ? c : best;
    }
    return best;
}
SS_HD int pool_table_cap(int aligned, const int* const* bounds, const int* N, const int* P, int n, int win_len, int K,
                         Block* full) {
    return pool_table_cap(aligned, bounds, N, P, nullptr, n, win_len, K, full);
}
// ---- trajectories of pooled slots (ss_trajectory, include/sonicsim_b200.h).  A slot with a trajectory reads, at every
// run, a path (a, b, dir) over its picked candidate's P positions and a bounds table of b - a + 1 entries, and renders the
// visited path: its local position j is bank position a + j (dir 0, forward) or b - j (dir 1, reverse), timed by the
// drawn bounds instead of the candidate's own.  Its counts block is 128 bytes: counts[25] bit 0 (written by the host)
// marks the trajectory, [28..29] and [30..31] hold the device pointers of its path and bounds.  The head of k_blocks
// (take_trajectory) runs after the pick: it shifts the slot's spectra (and cut table) to position a, takes the drawn
// bounds and P = b - a + 1, and sets counts[25] bit 1 for a reverse path.  h_rows keeps the bank's P*C*K: it is the
// offset of the direct set, which follows the same map.  A banked slot reads its cut table only as the mark of a direct
// set, so the cut table is shifted to position a whatever the direction.  The slot's work items are then filled by
// k_blocks itself, after its item scan (fill_traj_items): fill_items as k_prepare's range warps call it, and for a
// reverse path each item's RIR pointer moved to the last visited position with the position stride negated.  counts[0]
// is then set to 0, so that k_prepare's range warps leave the slot's items alone; its dry-window CTAs read the block
// table, not counts[0].  k_prepare is thus the parent's code for every source.  An invalid path (a >= b, a < 0,
// b > P - 1, dir not 0 or 1) or bounds table (not non-decreasing from 0 to N) leaves the candidate's own forward path and
// bounds, and the run reports kTrajBit.
constexpr unsigned kTrajBit = 256u;                    // bit 8 of ss_device_errors
SS_HD bool has_traj(const Source& s) { return s.h_rows && pool_table(s) && (s.counts[25] & 1); }
SS_HD const int* traj_path(const Source& s) { return *reinterpret_cast<const int* const*>(s.counts + 28); }
SS_HD const int* traj_bounds(const Source& s) { return *reinterpret_cast<const int* const*>(s.counts + 30); }
// a path (a, b, dir) over P positions and its bounds table b[0 .. b - a] of an N-sample candidate, as the slot takes them
SS_HD bool traj_valid(const int* path, const int* bounds, int P, int N) {
    const int a = path[0], b = path[1], dir = path[2];
    if (a < 0 || a >= b || b > P - 1 || (dir != 0 && dir != 1)) return false;
    if (bounds[0] != 0 || bounds[b - a] != N) return false;
    for (int q = 0; q < b - a; ++q) if (bounds[q + 1] < bounds[q]) return false;
    return true;
}
// The head of k_blocks for a slot with a trajectory, after the pick wrote the candidate into the slot's Source.  Returns
// the error bits to report.
SS_HD unsigned take_trajectory(Source& s) {
    const int* const path = traj_path(s);
    const int* const bounds = traj_bounds(s);
    s.counts[25] = 1;
    if (!traj_valid(path, bounds, s.P, s.N)) return kTrajBit;
    const int a = path[0];
    s.hspec += (size_t)a * s.C * s.K * kSpec;
    if (s.cut) s.cut += (size_t)a * s.C;
    s.bounds = bounds;
    s.P = path[1] - a + 1;
    s.counts[25] = 1 | (path[2] << 1);
    return 0;
}
// Table size of a slot with a trajectory: drawn bounds may cut blocks at other samples than any candidate's own, so
// under aligned blocking the table holds the blocks of any bounds table of at most P[i] - 1 segments over N[i] samples,
// at any start: the device-side bound of window_table_cap (at most ceil(o / 4096) + 1 blocks of each segment a window
// overlaps by o samples, one block in front and the last one's partner), never more than the whole candidate's
// table_cap (at most one partial block per segment).  Grid blocking does not read the bounds: pool_table_cap's.
SS_HD int traj_table_cap(int aligned, const int* N, const int* P, const int* Ks, int n, int win_len, int K, Block* full) {
    if (!aligned) return pool_table_cap(0, nullptr, N, P, Ks, n, win_len, K, full);
    int best = 0;
    for (int i = 0; i < n; ++i) {
        const int cap = table_cap(1, (N[i] + kB - 1) / kB, P[i]);
        const int c = window_table_cap(nullptr, 0, N[i], win_len, Ks ? Ks[i] : K, P[i], cap);
        best = c > best ? c : best;
    }
    return best;
}
// ---- host pools (SS_BANK_HOST, include/sonicsim_b200.h): banks and dry signals in pinned host memory.  At every run
// k_stage copies the read set of each pooled slot's picked candidate into the slot's staging area in device memory and
// writes the slot's view of it; the head of k_blocks then takes that view instead of the pool's entry.
// Read set of a window [ws, ws + len) of a candidate of N samples, P positions (bounds: its trajectory, unread when
// P == 1), C channels and K partitions - a superset of what k_blocks, k_prepare and the render kernels read:
//   - dry samples [xa, xb) = [ws - (K + 2) * 4096, ws + len + 2 * 4096) clamped to [0, N).  The table's first block g0
//     is at most K blocks in front of the block holding ws (window_span: K - 1 partition blocks, one more for the even
//     start) and starts after ws - (K + 1) * 4096; its dry window reaches 4096 further back.  The last block, the
//     partner of the last one that meets the window, starts before ws + len + 4096 and its window ends 4096 later.
//   - RIR rows [row0, row0 + rows) of each set: every position whose segment holds a sample of [xa, xb) and the one
//     after it (the blocks that meet the window lie inside [xa, xb)), widened to row pairs as window_rows does.
struct StageSet { int xa, xb, row0, rows; };
SS_HD StageSet stage_set(int N, int P, int C, int K, const int* bounds, int ws, int len) {
    StageSet r;
    const long long a = (long long)ws - (long long)(K + 2) * kB, b = (long long)ws + len + 2 * kB;
    r.xa = a > 0 ? (int)a : 0;
    r.xb = b < N ? (int)b : N;
    int pa = 0, pb = 0;
    if (P > 1) { pa = seg_of(bounds, P - 1, r.xa); pb = seg_of(bounds, P - 1, r.xb - 1) + 1; }
    window_rows(P, C, K, pa, pb, r.row0, r.rows);
    return r;
}
// Staging area of a pooled slot with windows of len over n candidates (candidate i: N[i], P[i], Ks[i] partitions,
// trajectory bounds[i], or bounds == null for a static pool): the most RIR rows per set and dry samples any candidate's
// read set holds at any start in [0, N[i] - len].  Both grow with the start while the first staged sample stays in one
// segment, so the rows are largest at the last start of each such run - stage_set at P[i] + 1 starts, O(P log P) per
// candidate - and the dry span at min(N[i] - len, (K + 2) * 4096).  The dry count has 8 samples to spare: k_stage
// copies whole float4s around the read set.
SS_HD void stage_cap(const int* const* bounds, const int* N, const int* P, const int* Ks, int n, int C, int len,
                     int& rows, int& nx) {
    rows = 0; nx = 0;
    for (int i = 0; i < n; ++i) {
        const int last = N[i] - len;
        const long long d0 = (long long)(Ks[i] + 2) * kB;
        const int* const b = bounds ? bounds[i] : nullptr;
        for (int sg = -2; sg < (b ? P[i] - 1 : 0); ++sg) {
            // the last start, the widest dry span, then the last start of each segment's run
            const long long w = sg == -2 ? last : sg == -1 ? d0 : b[sg + 1] - 1 + d0;
            const StageSet r = stage_set(N[i], P[i], C, Ks[i], b, w < last ? (int)w : last, len);
            rows = r.rows > rows ? r.rows : rows;
            nx = r.xb - r.xa + 8 > nx ? r.xb - r.xa + 8 : nx;
        }
    }
}
// A slot's view of its picked candidate, written by k_stage: the pool's entry with x (biased: sample n at x[n]) and spec
// pointing into the staging area, whose sets hold rows [row0, row0 + rows) back to back; the candidate's K and gain.
struct StageView {
    PoolEntry e;
    int K, row0, rows;
    float gain;
};
static_assert(sizeof(StageView) == 56, "StageView layout");
// A pooled slot's counts[18..19]: the device pointer of its StageView (a slot of a host pool), or null
SS_HD const StageView* stage_view(const Source& s) { return *reinterpret_cast<const StageView* const*>(s.counts + 18); }
// The head of k_blocks for a slot of a host pool: the staged view into the slot's Source, as pick_slot writes an entry of a
// device pool, with the staged rows as the window's row origin (h_row0, h_rows; fill_items addresses rows through it)
SS_HD void take_view(Source& s, const StageView& v) {
    s.K = v.K;
    pick_candidate(s, v.e);
    s.h_row0 = v.row0; s.h_rows = v.rows;
    set_stem_gain(s, v.gain);
}
// ---- dry pools (ss_dry_pool, include/sonicsim_b200.h).  A dry-picked slot of a device pool renders its picked
// candidate with the dry signal its own pick names in a dry pool.  Its counts block is 112 bytes, as every pooled slot's:
// [20..21] the device pointer of the dry pool's n signal pointers, or null (no dry pick), [22..23] the device pointer of
// the dry pick, [24] the dry pool's signal count, [26..27] the device pointer of the slot's pair gains (ss_pair_gains),
// or null.
SS_HD const float* const* dry_table(const Source& s) { return *reinterpret_cast<const float* const* const*>(s.counts + 20); }
SS_HD const int* dry_pick_ptr(const Source& s) { return *reinterpret_cast<const int* const*>(s.counts + 22); }
SS_HD int dry_size(const Source& s) { return s.counts[24]; }
SS_HD const float* pair_table(const Source& s) { return *reinterpret_cast<const float* const*>(s.counts + 26); }
// The dry pick v read from device memory, clamped into [0, n) (bad = it was not there): the picked signal replaces the
// candidate's own x.  Everything else - N, P, bounds, K, spectra, cuts, gain - stays the trajectory candidate's, and only
// samples [0, N) of x are read, so a dry signal at least N long renders as that candidate with the signal's first N.
// Returns the clamped pick.
SS_HD int pick_dry(Source& s, int v, bool& bad) {
    const int d = clamp_pick(v, dry_size(s), bad);
    s.x = dry_table(s)[d];
    return d;
}
// Pair gains (ss_pair_gains): the (float)gain of dry signal d through candidate i of a pool of n, measured on the pair's
// whole stem; it replaces the candidate's own gain
SS_HD float pair_gain(const float* table, int d, int i, int n) { return table[(long long)d * n + i]; }
// The head of k_blocks for a pooled slot of a device pool: the trajectory pick (its K, then its candidate and gain), then
// the dry pick of a dry-picked slot, and with pair gains the pair's gain.  Returns the error bits to report: 8 for a
// clamped pick, 16 for a clamped dry pick.
SS_HD unsigned pick_pooled(Source& s) {
    bool bad;
    unsigned err = 0;
    const int v = *pick_ptr(s);
    pick_parts(s, v);                       // the picked candidate's K first: set_banked reads it
    pick_slot(s, v, bad);
    if (bad) err |= 8u;
    if (dry_table(s)) {
        const int d = pick_dry(s, *dry_pick_ptr(s), bad);
        if (bad) err |= 16u;
        if (const float* const t = pair_table(s))
            set_stem_gain(s, pair_gain(t, d, clamp_pick(v, pool_size(s), bad), pool_size(s)));
    }
    return err;
}
// The head of k_stage for one staged slot (a slot of a host pool, or a slot with a dry pick from a host dry pool): the
// pick (clamped into [0, n), bit 3), the picked candidate's K (parts[i], or K) and start (ws_dev's, clamped - bit 2 is
// k_blocks' - or ws), its read set (stage_set) and the view the head of k_blocks takes.  A slot of a host pool (rows)
// stages rows [row0, row0 + rows) of each set; a slot of a device pool keeps its bank's spectra, row0 = 0 and rows =
// P*C*K, what set_banked gives it.  A dry-picked slot (dry: the dry pool's signal table, in mapped host memory) then
// reads its dry pick (clamped into [0, n_dry), bit 16) and stages that signal's samples instead of the candidate's x:
// the read set stays the candidate's, inside [0, N).  With pair gains (pair: a dry-picked slot's table) the view takes
// the pair's gain in place of the candidate's.  src receives the signal to copy, [x0, x1) the whole float4s around
// [xa, xb) (a host arena pads every signal to whole float4s).  Returns the error bits.
SS_HD unsigned stage_head(const PoolEntry* pool, int n, int v, const int* parts, int K, const float* gains,
                          const int* ws_dev, int ws, int len, int C, bool rows, const float* const* dry, int dv,
                          int n_dry, StageView& view, const float*& src, int& x0, int& x1, const float* pair = nullptr) {
    bool bad;
    unsigned err = 0;
    const int i = clamp_pick(v, n, bad);
    if (bad) err |= 8u;
    const PoolEntry e = pool[i];
    const int k = parts ? parts[i] : K;
    if (ws_dev) ws = clamp_win_start(*ws_dev, e.N, len, bad);
    const StageSet r = stage_set(e.N, e.P, C, k, e.bounds, ws, len);
    view.e = e; view.K = k; view.gain = gains ? gains[i] : 1.0f;
    view.row0 = rows ? r.row0 : 0;
    view.rows = rows ? r.rows : e.P * C * k;
    src = e.x;
    if (dry) {
        const int d = clamp_pick(dv, n_dry, bad);
        src = dry[d];
        if (bad) err |= 16u;
        if (pair) view.gain = pair_gain(pair, d, i, n);
    }
    x0 = r.xa & ~3; x1 = (r.xb + 3) & ~3;
    return err;
}
// ---- crop start draws of device plans (ss_plan_draw, include/sonicsim_b200.h): the dataloader's start loop
// (movingdatamodule.py:81-99) over level tables Q (ss_pool_levels: Q[0] = 0, Q[n + 1] = Q[n] + e[n], float64).
// Starts a crop of len samples can take in a candidate of N samples: the M of a draw is the least of these over its readers
SS_HD int draw_span(int N, int len) { return N - len + 1; }
// Try t's start: min(floor(u * M), M - 1), in float64 (randint(0, M - 1) with its uniform variate given); a u outside
// [0, 1) maps into range: u >= 1 to M - 1, u < 0 or NaN to 0
SS_HD int draw_start(double u, int M) {
    const double v = floor(u * (double)M);
    if (!(v > 0.0)) return 0;
    return v < (double)(M - 1) ? (int)v : M - 1;
}
// compute_mch_rms_dB (:29-32) of the crop [s, s + len) of a table below the threshold: silent.  D = len (mono table) or
// C * len (channel table): the crop's element count
SS_HD bool draw_silent_sums(double q0, double q1, double D, float threshold_db) {
    double ms = (q1 - q0) / D;
    if (ms < 1e-20) ms = 1e-20;
    return 10.0 * log10(ms) < (double)threshold_db;
}
SS_HD bool draw_silent(const double* Q, int s, int len, double D, float threshold_db) {
    const double q1 = Q[s + len];
    return draw_silent_sums(Q[s], q1, D, threshold_db);
}
// ---- 16-bit dry pools (ss_dry_pool_create_i16): sample k of a signal stands for k / 32768, exactly a float32.  Its
// float32 square is a multiple of 2^-30 and at most 1, so for N <= 2^23 every partial sum of the level table is a
// multiple of 2^-30 below 2^53 * 2^-30: exact in float64, whatever the order of the sum.  The pool keeps the table at
// stride kLevelStride, q[j] = Q[min(64 j, N)] for j = 0..ceil(N / 64), and any Q[s] is q[s / 64] plus the exact sum of
// the at most 63 squares behind it: bit for bit the full table's entry.
constexpr int kLevelStride = 64;
SS_HD float i16_sample(int16_t v) { return (float)v * (1.0f / 32768.0f); }
// four samples of a 16-bit signal as k_stage stores them into a staging area of float32 samples
SS_HD float4 i16x4_samples(short4 v) {
    return make_float4(i16_sample(v.x), i16_sample(v.y), i16_sample(v.z), i16_sample(v.w));
}
// Q[s] (0 <= s <= N) of a 16-bit signal x from its sparse table q
SS_HD double sparse_level(const double* q, const int16_t* x, int s) {
    const int j = s / kLevelStride;
    double a = q[j];
    for (int n = j * kLevelStride; n < s; ++n) {
        const float v = i16_sample(x[n]);
        a += (double)(v * v);                           // the term k_levels adds
    }
    return a;
}
// draw_silent of a 16-bit dry-picked speaker (D = len)
SS_HD bool draw_silent_i16(const double* q, const int16_t* x, int s, int len, float threshold_db) {
    return draw_silent_sums(sparse_level(q, x, s), sparse_level(q, x, s + len), (double)len, threshold_db);
}
// The level table a draw tests for one speaker: a dry-picked speaker's (dry_levels non-null) is its dry pool's table of
// the picked dry signal, whose crops have D = len; any other's is its pool's table of the picked candidate.  Both picks
// are clamped as k_blocks clamps them.
SS_HD const double* speaker_table(const double* const* levels, const int* pick, int n, const double* const* dry_levels,
                                  const int* dry_pick, int n_dry) {
    bool bad;
    return dry_levels ? dry_levels[clamp_pick(*dry_pick, n_dry, bad)] : levels[clamp_pick(*pick, n, bad)];
}
// The picked signal of a dry-picked speaker whose dry pool is 16-bit, clamped as speaker_table clamps it: such a pool's
// device pointer array holds its n_dry signal pointers and then its n_dry table pointers, dry_levels.
SS_HD const int16_t* speaker_signal_i16(const double* const* dry_levels, const int* dry_pick, int n_dry) {
    bool bad;
    return reinterpret_cast<const int16_t* const*>(dry_levels - n_dry)[clamp_pick(*dry_pick, n_dry, bad)];
}
// ---- dry streams (ss_dry_stream, include/sonicsim_b200.h): a stream slot's dry signal is laid out at every run from
// m (ids, offsets) entries over a 16-bit dry pool of n utterances.  The walk: an entry with id < 0 is empty and
// skipped; one with id >= n, offset < 0 or offset < end (the end of the last kept entry, 0 at first) is invalid,
// skipped and reported (bit 5); any other is kept: utterance id of len samples occupies [offset, offset + len) of the
// stream and end becomes offset + len.  Zeros lie wherever no kept entry does.  k_stage, k_draw and the CPU emulation
// decide validity through this one walk (layout_entries), which background streams (ss_bg_stream, bg_entries) share:
// a speech stream is the bed form with head 0 and count len.
constexpr int kStreamEntries = 128;                    // the most entries of a layout
constexpr unsigned kStreamBit = 32u;                   // bit 5 of ss_device_errors: an invalid entry was skipped
// Walks entries [0, m) of a layout over n clips: span(j, id, head, count) sets the clip samples [head, head + count)
// entry j places (id valid) and returns false when they are not a non-empty range of the clip (an invalid entry);
// kept(j, id, offset, head, count) sees each kept entry in order and returns false to end the walk there.  Returns
// kStreamBit if an invalid entry was met.
template <class Span, class Kept>
SS_HD unsigned layout_entries(const int* ids, const int* offsets, int m, int n, Span span, Kept kept) {
    unsigned err = 0;
    long long end = 0;
    for (int j = 0; j < m; ++j) {
        const int id = ids[j];
        if (id < 0) continue;
        const int o = offsets[j];
        if (id >= n || o < 0 || o < end) { err = kStreamBit; continue; }
        int head, count;
        if (!span(j, id, head, count)) { err = kStreamBit; continue; }
        end = (long long)o + count;
        if (!kept(j, id, o, head, count)) break;
    }
    return err;
}
// A speech stream's walk: len_of(j, id) gives the length of entry j's utterance (id valid), kept(j, id, offset, len)
// sees each kept entry in order and returns false to end the walk there.  Returns kStreamBit if an invalid entry was
// met.
template <class Len, class Kept>
SS_HD unsigned stream_entries(const int* ids, const int* offsets, int m, int n, Len len_of, Kept kept) {
    return layout_entries(ids, offsets, m, n,
                          [&](int j, int id, int& head, int& count) { head = 0; count = len_of(j, id); return true; },
                          [&](int j, int id, int o, int, int count) { return kept(j, id, o, count); });
}
// A background stream's walk: entry j places clip samples [heads[j], heads[j] + counts[j]), which must lie in the clip
// of len_of(j, id) samples with counts[j] >= 1; kept as for layout_entries.
template <class Len, class Kept>
SS_HD unsigned bg_entries(const int* ids, const int* offsets, const int* heads, const int* counts, int m, int n,
                          Len len_of, Kept kept) {
    return layout_entries(ids, offsets, m, n,
                          [&](int j, int id, int& head, int& count) {
                              head = heads[j]; count = counts[j];
                              return head >= 0 && count >= 1 && (long long)head + count <= len_of(j, id);
                          },
                          kept);
}
// The kept entry covering stream sample n of a resolved layout whose k entries start at a[] ascending, plus one: 0 when
// none starts at or before n (the caller tests n < b[lo - 1])
SS_HD int layout_find(const int* a, int k, int n) {
    int lo = 0, hi = k;                                 // the first entry starting after n
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (a[mid] <= n) lo = mid + 1; else hi = mid;
    }
    return lo;
}
// A stream slot's descriptor in its plan's block (the plan's copy of its dry pool's utterance lengths, the pool's
// signal and sparse-table pointers - ss_dry_pool::ptrs); cut is the slot pool's longest N, the length of the stream a
// DryPick of the same layout would pick from a 16-bit pool.
struct DryStream {
    const int* ids;
    const int* offsets;
    const int* lengths;
    const int16_t* const* sig;
    const double* const* levels;                       // null without level tables
    int m, n, cut, pad;
};
static_assert(sizeof(DryStream) == 56, "DryStream layout");
// The kept entries of a layout cut at `cut`, for per-sample lookups (stream_sample): a[k] <= n < b[k] is covered by
// utterance p[k] at sample n - a[k], k ascending in a.  len[j] is entry j's utterance length (read where its id is
// valid) and sig[j] its signal.  *count receives the number of entries; returns stream_entries' error bits.
SS_HD unsigned stream_resolve(const int* ids, const int* offsets, const int* len, const int16_t* const* sig, int m,
                              int n, int cut, int* a, int* b, const int16_t** p, int* count) {
    int k = 0;
    const unsigned err = stream_entries(ids, offsets, m, n, [&](int j, int) { return len[j]; },
                                        [&](int j, int, int o, int l) {
                                            if (o < cut) {       // (an entry at or past the cut adds no sample)
                                                const long long e = (long long)o + l;
                                                a[k] = o; b[k] = e < cut ? (int)e : cut; p[k] = sig[j];
                                                ++k;
                                            }
                                            return true;
                                        });
    *count = k;
    return err;
}
// Sample n of a resolved stream (stream_resolve: k entries), as k_stage stores it: the covering utterance's sample
// (i16_sample), or 0
SS_HD float stream_sample(const int* a, const int* b, const int16_t* const* p, int k, int n) {
    const int lo = layout_find(a, k, n);
    return lo > 0 && n < b[lo - 1] ? i16_sample(p[lo - 1][n - a[lo - 1]]) : 0.0f;
}
// The energy of the crop [s, s + len) of a stream (s + len at most the stream's cut): over the kept entries that meet
// it, the utterance-local differences of sparse_level.  Every term is a multiple of 2^-30 and the sum stays below 2^23
// (the crop's squares are at most 1 each), so the sum is exact in float64 in any order: Q[s + len] - Q[s] of the
// assembled stream's full table, bit for bit.
SS_HD double stream_level(const DryStream& d, int s, int len) {
    double q = 0.0;
    const long long lo = s, hi = (long long)s + len;
    stream_entries(d.ids, d.offsets, d.m, d.n, [&](int, int id) { return d.lengths[id]; },
                   [&](int, int id, int o, int l) {
                       if (o >= hi) return false;       // (later entries start later still)
                       const long long b0 = lo > o ? lo - o : 0, b1 = hi - o < l ? hi - o : l;
                       if (b1 > b0)
                           q += sparse_level(d.levels[id], d.sig[id], (int)b1) -
                                sparse_level(d.levels[id], d.sig[id], (int)b0);
                       return true;
                   });
    return q;
}
// draw_silent of a stream speaker (D = len)
SS_HD bool draw_silent_stream(const DryStream& d, int s, int len, float threshold_db) {
    return draw_silent_sums(0.0, stream_level(d, s, len), (double)len, threshold_db);
}
// ---- background streams (ss_bg_stream, include/sonicsim_b200.h): a bed slot's dry signal is laid out at every run
// from m (ids, offsets, heads, counts) entries over a dry pool of n clips, float32 or 16-bit (bg_entries' walk).
// A bed slot's descriptor in its plan's block: the layout, the plan's copy of the clip lengths and the pool's signal
// pointers (float or int16 addresses, i16 telling which); cut as for DryStream.
struct BgStream {
    const int* ids;
    const int* offsets;
    const int* heads;
    const int* counts;
    const int* lengths;
    const char* const* sig;
    int m, n, cut, i16;
};
static_assert(sizeof(BgStream) == 64, "BgStream layout");
// The kept entries of a bed layout cut at `cut`, as stream_resolve resolves a speech stream's: a[k] <= n < b[k] is
// covered by element n - a[k] of p[k], the clip's address sig[j] advanced by its head (elements of `size` bytes).
// len[j] is entry j's clip length (read where its id is valid).
SS_HD unsigned bg_resolve(const int* ids, const int* offsets, const int* heads, const int* counts, const int* len,
                          const char* const* sig, int size, int m, int n, int cut, int* a, int* b, const char** p,
                          int* count) {
    int k = 0;
    const unsigned err = bg_entries(ids, offsets, heads, counts, m, n, [&](int j, int) { return len[j]; },
                                    [&](int j, int, int o, int h, int c) {
                                        if (o < cut) {
                                            const long long e = (long long)o + c;
                                            a[k] = o; b[k] = e < cut ? (int)e : cut; p[k] = sig[j] + (size_t)h * size;
                                            ++k;
                                        }
                                        return true;
                                    });
    *count = k;
    return err;
}
// Sample n of a resolved bed (bg_resolve: k entries), as k_stage stores it: the covering clip's sample (an int16 clip's
// through i16_sample), or 0
SS_HD float bg_sample(const int* a, const int* b, const char* const* p, int k, int n, bool i16) {
    const int lo = layout_find(a, k, n);
    if (lo == 0 || n >= b[lo - 1]) return 0.0f;
    const int t = n - a[lo - 1];
    return i16 ? i16_sample(reinterpret_cast<const int16_t*>(p[lo - 1])[t]) : reinterpret_cast<const float*>(p[lo - 1])[t];
}

// ---- layout draws (ss_layout_draw, include/sonicsim_b200.h): a plan draws a stream or bed slot's layout itself at
// every run (k_layout), from a counter-based generator, by the rules of dry.long_audio_layouts and
// dry.background_audio_layouts.  The random stream is a format: the kernel, the CPU emulation and the tests' Python
// restatement follow it word for word.
//   - Philox4x32-10 (Salmon et al., SC'11), written out here so that g++ compiles it for the emulation.
//   - The key is the 64-bit seed (seed_lo, seed_hi).  Block b of layout draw r (its index in the plan's list of draws)
//     at counter t is philox(ctr = (b, r, t_lo, t_hi), key), b = 0, 1, ...; its 4 words are consumed in order.
//   - A uniform integer in [0, k) takes the next two words, x = w0 | w1 << 32, and is umulhi64(x, k).
// (seed, t) are two int64 in device memory, read at every run: the same pair draws the same layouts, bit for bit.
constexpr int kLayoutCap = 1024;                       // the most utterances or clips one row may select
SS_HD uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
    for (int i = 0; i < 10; ++i) {
        if (i) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
        const uint64_t p0 = (uint64_t)0xD2511F53u * c.x, p1 = (uint64_t)0xCD9E8D57u * c.z;
        c = make_uint4((uint32_t)(p1 >> 32) ^ c.y ^ k0, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ k1, (uint32_t)p0);
    }
    return c;
}
SS_HD uint64_t umulhi64(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    return __umul64hi(a, b);
#else
    return (uint64_t)(((unsigned __int128)a * b) >> 64);
#endif
}
// The word stream of one layout draw at one (seed, t)
struct LayoutRng {
    uint32_t k0, k1, r, t0, t1, b;
    int w;                                             // words of buf consumed
    uint4 buf;
};
SS_HD LayoutRng layout_rng(int64_t seed, int64_t t, int r) {
    LayoutRng g;
    g.k0 = (uint32_t)(uint64_t)seed; g.k1 = (uint32_t)((uint64_t)seed >> 32);
    g.r = (uint32_t)r; g.t0 = (uint32_t)(uint64_t)t; g.t1 = (uint32_t)((uint64_t)t >> 32);
    g.b = 0; g.w = 4; g.buf = make_uint4(0, 0, 0, 0);
    return g;
}
SS_HD uint32_t rng_word(LayoutRng& g) {
    if (g.w == 4) { g.buf = philox4x32_10(make_uint4(g.b++, g.r, g.t0, g.t1), g.k0, g.k1); g.w = 0; }
    const int w = g.w++;
    return w == 0 ? g.buf.x : w == 1 ? g.buf.y : w == 2 ? g.buf.z : g.buf.w;
}
// a uniform integer in [0, k), k >= 1
SS_HD uint64_t rng_below(LayoutRng& g, uint64_t k) {
    const uint64_t lo = rng_word(g);
    return umulhi64(lo | (uint64_t)rng_word(g) << 32, k);
}
// One layout draw's descriptor in its plan's block.  heads == null: a speech stream (create_long_audio's rule), else a
// bed (create_background_audio's).  lengths: the plan's copy of the dry pool's n lengths; select: a bed's n selection
// lengths, or null for the lengths themselves.  K (<= kLayoutCap) bounds what a row can select: the scratch of a row is
// a hash map of map_cap (a power of two >= 2K + 2) keys and values and K selected ids.
struct LayoutDesc {
    const int64_t* rng;
    const int* lengths;
    const int* select;
    int* ids;
    int* offsets;
    int* heads;
    int* counts;
    int n, m, total, gap_max, K, r, map_cap, pad;
};
static_assert(sizeof(LayoutDesc) == 88, "LayoutDesc layout");
SS_HD int layout_map_cap(int K) { int c = 2; while (c < 2 * K + 2) c <<= 1; return c; }
SS_HD int layout_scratch_ints(int K) { return 2 * layout_map_cap(K) + K; }
// The sparse Fisher-Yates array: position i holds the map's value for key i, or i itself (keys -1: empty slots)
SS_HD unsigned fy_slot(int i, int mask) { return ((uint32_t)i * 2654435769u >> 7) & (unsigned)mask; }
SS_HD int fy_get(const int* keys, const int* vals, int mask, int i) {
    for (unsigned h = fy_slot(i, mask);; h = (h + 1) & (unsigned)mask) {
        if (keys[h] == i) return vals[h];
        if (keys[h] < 0) return i;
    }
}
SS_HD void fy_put(int* keys, int* vals, int mask, int i, int v) {
    for (unsigned h = fy_slot(i, mask);; h = (h + 1) & (unsigned)mask)
        if (keys[h] == i || keys[h] < 0) { keys[h] = i; vals[h] = v; return; }
}
// One row, in the order its words are drawn (keys: map_cap entries of -1; vals: map_cap; sel: K):
//   1. selection, a uniform order over the n ids without replacement (step s swaps position s with s + u, u uniform
//      in [0, n - s)): a stream takes the drawn utterance while the running total is below 0.9 * total and stops at the
//      first that would overflow `total` (get_random_wav_path); a bed takes clips while the running total of `select`
//      is below 0.4 * total, and the clip that reaches `total` is taken and ends it (get_random_wav_path_from_json);
//   2. placement, the selected ids in a fresh uniform order (step j swaps j with j + v, v uniform in [0, s - j)) while
//      the cursor is below `total`, each followed by one more draw: a stream's gap in {0, ..., gap_max} before the
//      utterance, placed while cursor + gap + len <= total (_place_long_audio); a bed's tail in {0, ..., gap_max} after
//      the clip, and the first clip with len + tail >= total - cursor is the end clip: slack = floor((total - cursor) *
//      0.1), lead and trail uniform in {0, ..., slack}, kept with head lead and count min(len, total - trail - cursor) -
//      lead when that is above 0 (_place_background_audio);
//   3. the first m entries in stream order, then -1 in every array.
SS_HD void layout_row(const LayoutDesc& d, int* keys, int* vals, int* sel) {
    LayoutRng g = layout_rng(d.rng[0], d.rng[1], d.r);
    const int mask = d.map_cap - 1;
    const bool bed = d.heads != nullptr;
    const int* const sl = d.select ? d.select : d.lengths;
    const double thr = (bed ? 0.4 : 0.9) * (double)d.total;
    long long acc = 0;
    int s = 0;
    while (s < d.n && (double)acc < thr) {
        const int p = s + (int)rng_below(g, (uint64_t)(d.n - s));
        const int x = fy_get(keys, vals, mask, p);
        const long long l = sl[x];
        if (!bed && acc + l > d.total) break;
        if (s == d.K) break;                           // (never: K bounds every selection)
        fy_put(keys, vals, mask, p, fy_get(keys, vals, mask, s));
        sel[s++] = x;
        if (bed && !(acc + l < d.total)) break;
        acc += l;
    }
    long long cur = 0;
    int k = 0;
    auto put = [&](int id, long long o, long long h, long long c) {
        d.ids[k] = id; d.offsets[k] = (int)o;
        if (bed) { d.heads[k] = (int)h; d.counts[k] = (int)c; }
        ++k;
    };
    for (int j = 0; j < s && cur < d.total && k < d.m; ++j) {
        const int v = j + (int)rng_below(g, (uint64_t)(s - j));
        const int id = sel[v];
        sel[v] = sel[j]; sel[j] = id;
        const long long l = d.lengths[id];
        const long long gap = (long long)rng_below(g, (uint64_t)d.gap_max + 1);
        if (!bed) {
            if (cur + gap + l > d.total) break;
            put(id, cur + gap, 0, l);
            cur += gap + l;
        } else if (l + gap >= d.total - cur) {
            const long long slack = (long long)floor((double)(d.total - cur) * 0.1);
            const long long lead = (long long)rng_below(g, (uint64_t)slack + 1);
            const long long trail = (long long)rng_below(g, (uint64_t)slack + 1);
            const long long c = (l < d.total - trail - cur ? l : d.total - trail - cur) - lead;
            if (c > 0) put(id, cur + lead, lead, c);
            break;
        } else {
            put(id, cur, 0, l);
            cur += l + gap;
        }
    }
    for (; k < d.m; ++k) {
        d.ids[k] = -1; d.offsets[k] = -1;
        if (bed) { d.heads[k] = -1; d.counts[k] = -1; }
    }
}

// ---- grouped layout draws (ss_layout_group, include/sonicsim_b200.h): a stream slot's draw over one of G >= 1
// contiguous groups of its pool's utterances, 0 = b[0] < b[1] < ... < b[G] = n (e.g. one LibriSpeech speaker's
// utterances each, as SonicSet builds every stream from one speaker), the group g read from device memory at every run.
//   - g outside [0, G) is clamped into range and the run reports bit 7 (ss_device_errors);
//   - the row is then exactly the ungrouped draw r over a pool holding only utterances [b[g], b[g + 1]), in order: the
//     same Philox blocks (b, r, t_lo, t_hi), the same words in the same order; every id it writes is offset by b[g];
//   - reading g consumes no words.
// So G = 1 is the ungrouped draw, and group g over the whole pool is the ungrouped draw over that group's sub-pool with
// its ids shifted.  K of a grouped draw is the largest K of its groups (a larger K than a group's own changes none of
// its words: the bound is never reached).
struct LayoutGroup {
    const int* group;                                  // device, one int32 read at every run; null: an ungrouped draw
    const int* bounds;                                 // the plan's copy of the G + 1 bounds
    int G, pad;
};
static_assert(sizeof(LayoutGroup) == 24, "LayoutGroup layout");
// The row of layout draw d under its group entry q (q.group null: layout_row's row itself); returns the error bits
SS_HD unsigned layout_row_grouped(LayoutDesc d, const LayoutGroup& q, int* keys, int* vals, int* sel) {
    unsigned err = 0;
    int lo = 0;
    if (q.group) {                                     // narrow the pool to the group's utterances
        int g = *q.group;
        if (g < 0 || g >= q.G) {
            g = g < 0 ? 0 : q.G - 1;
            err = 128u;
        }
        lo = q.bounds[g];
        d.lengths += lo;
        d.n = q.bounds[g + 1] - lo;
    }
    layout_row(d, keys, vals, sel);
    if (lo)
        for (int k = 0; k < d.m; ++k)
            if (d.ids[k] != -1) d.ids[k] += lo;
    return err;
}

// ---- value draws (ss_value_draw, include/sonicsim_b200.h): a plan writes the per-run values its slots, draws,
// mixtures and loudness slots read (picks, starts, SIRs, SNRs, crop variates, loudness targets) itself at the head of
// every run (k_values), from the generator of the layout draws.  The random stream is a format, followed word for word
// by the kernel, the CPU emulation and the tests' Python restatement:
//   - the key is the 64-bit seed (seed_lo, seed_hi), as for layout draws;
//   - element j of row b of value draw r (its index in the plan's list of value draws) at counter t takes block
//     philox(ctr = (b, 0x80000000 | r << 11 | j >> 1, t_lo, t_hi), key) and its words 2 (j & 1) and 2 (j & 1) + 1 as
//     x = w0 | w1 << 32.  Layout draws use c1 = r < 2^31, so the two streams never share a block (r < 2^20, k <= 4096);
//   - float64: u = (x >> 11) * 2^-53; float32: u = (x >> 40) * 2^-24; v = low + (high - low) * u in float64 (product
//     and sum rounded separately), rounded once to the output type; a result not below high becomes the largest value
//     of the type below high;
//   - int32: low + umulhi64(x, high - low);
//   - distinct: a partial Fisher-Yates over [0, n), n = high - low: element j takes y = umulhi64(x_j, n - j) and
//     pos = j + y, writes low + a[pos] and sets a[pos] = a[j] (a: the identity, held as a sparse map);
//   - with a base draw, the value is base[b] * stride + value (int64; creation rules out int32 overflow).
// Every element is independent of the others except within a distinct row.
enum { VALUE_F32 = 0, VALUE_F64 = 1, VALUE_INT = 2, VALUE_DISTINCT = 3 };
constexpr int kValueDrawsMax = 1 << 20;                // r < 2^20: r << 11 stays below bit 31
constexpr int kValueMapCap = 128;                      // sparse Fisher-Yates map of a distinct row: >= 2k keys, k <= 64
struct ValueDesc {
    void* out;                                         // rows x k elements of the kind's type
    const int64_t* rng;                                // (seed, t)
    const int* base;                                   // int kinds: the (rows,) out of an earlier draw, or null
    double low, high;                                  // real kinds
    int ilow;                                          // int kinds: low
    uint32_t n;                                        // int kinds: high - low
    int kind, k, r, stride;
};
static_assert(sizeof(ValueDesc) == 64, "ValueDesc layout");
SS_HD uint64_t value_word(uint32_t k0, uint32_t k1, uint32_t t0, uint32_t t1, int r, int b, int j) {
    const uint4 w = philox4x32_10(make_uint4((uint32_t)b, 0x80000000u | (uint32_t)r << 11 | (uint32_t)j >> 1, t0, t1),
                                  k0, k1);
    return (j & 1) ? (w.z | (uint64_t)w.w << 32) : (w.x | (uint64_t)w.y << 32);
}
// low + (high - low) * u, the product and the sum each rounded once
SS_HD double value_lerp(double low, double high, double u) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(low, __dmul_rn(high - low, u));
#else
    return low + (high - low) * u;
#endif
}
// The float64 and the float32 value of word x in [low, high)
SS_HD double value_f64(double low, double high, uint64_t x) {
    const double v = value_lerp(low, high, (double)(x >> 11) * 0x1p-53);
    return v < high ? v : nextafter(high, -(double)INFINITY);
}
SS_HD float value_f32(double low, double high, uint64_t x) {
    const float v = (float)value_lerp(low, high, (double)(x >> 40) * 0x1p-24);
    return v < (float)high ? v : nextafterf((float)high, -INFINITY);
}
SS_HD unsigned vmap_slot(uint32_t i) { return (i * 2654435769u) >> 25; }   // 7 bits: kValueMapCap slots
SS_HD uint32_t vmap_get(const uint32_t* keys, const uint32_t* vals, uint32_t i) {
    for (unsigned h = vmap_slot(i);; h = (h + 1) & (kValueMapCap - 1)) {
        if (keys[h] == i) return vals[h];
        if (keys[h] == 0xFFFFFFFFu) return i;
    }
}
SS_HD void vmap_put(uint32_t* keys, uint32_t* vals, uint32_t i, uint32_t v) {
    for (unsigned h = vmap_slot(i);; h = (h + 1) & (kValueMapCap - 1))
        if (keys[h] == i || keys[h] == 0xFFFFFFFFu) { keys[h] = i; vals[h] = v; return; }
}
// Row b of value draw d: lane `lane` of `lanes` writes elements lane, lane + lanes, ...; a distinct row is drawn by
// lane 0 alone over the kValueMapCap keys and values of its map (the others return).  A base draw's row b must be
// written and visible before this call.
SS_HD void value_row(const ValueDesc& d, int b, int lane, int lanes, uint32_t* keys, uint32_t* vals) {
    const uint64_t seed = (uint64_t)d.rng[0], t = (uint64_t)d.rng[1];
    const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32), t0 = (uint32_t)t, t1 = (uint32_t)(t >> 32);
    const size_t row = (size_t)b * d.k;
    if (d.kind == VALUE_F32 || d.kind == VALUE_F64) {
        for (int j = lane; j < d.k; j += lanes) {
            const uint64_t x = value_word(k0, k1, t0, t1, d.r, b, j);
            if (d.kind == VALUE_F64) static_cast<double*>(d.out)[row + j] = value_f64(d.low, d.high, x);
            else static_cast<float*>(d.out)[row + j] = value_f32(d.low, d.high, x);
        }
        return;
    }
    const int64_t add = (int64_t)d.ilow + (d.base ? (int64_t)d.base[b] * d.stride : 0);
    int* const out = static_cast<int*>(d.out) + row;
    if (d.kind == VALUE_INT) {
        for (int j = lane; j < d.k; j += lanes)
            out[j] = (int)(add + (int64_t)umulhi64(value_word(k0, k1, t0, t1, d.r, b, j), d.n));
        return;
    }
    if (lane) return;
    for (int i = 0; i < kValueMapCap; ++i) keys[i] = 0xFFFFFFFFu;
    for (int j = 0; j < d.k; ++j) {
        const uint32_t pos = (uint32_t)j + (uint32_t)umulhi64(value_word(k0, k1, t0, t1, d.r, b, j), d.n - (uint32_t)j);
        out[j] = (int)(add + vmap_get(keys, vals, pos));
        vmap_put(keys, vals, pos, vmap_get(keys, vals, (uint32_t)j));
    }
}

// blocks of the table that meet the window: [win_first(s), win_first(s) + win_blocks(s)); all of them when unwindowed
SS_HD int win_first(const Source& s) { return s.h_rows ? s.counts[2] : 0; }
SS_HD int win_blocks(const Source& s) { return s.h_rows ? s.counts[3] : s.counts[0]; }

// Position range of a block (k_prepare's range warps).  Indexed source: block_pos_scan gives lane `lane` of `nlanes` the
// min / max of idx over its share of the block's samples; block_positions takes the combined [pmin, pmax].
SS_HD void block_pos_scan(const Source& S, const Block& bk, int lane, int nlanes, int& pmin, int& pmax) {
    pmin = 0x7fffffff; pmax = -1;
    for (int n = bk.start + lane; n < bk.start + bk.len; n += nlanes) { int v = S.idx[n]; pmin = v < pmin ? v : pmin; pmax = v > pmax ? v : pmax; }
}
// the positions block bk interpolates between: from the bounds (grid blocking), [pmin, pmax + 1] clamped to
// [0, P - 1] (indexed), as planned otherwise (aligned blocking, static source)
SS_HD Block block_positions(const Source& S, Block bk, int pmin, int pmax) {
    if (S.mode == MODE_MOVING_BOUNDS && !S.aligned) {
        bk.p_lo = seg_of(S.bounds, S.P - 1, bk.start);
        bk.p_hi = seg_of(S.bounds, S.P - 1, bk.start + bk.len - 1) + 1;
    } else if (S.mode == MODE_MOVING_INDEXED) {
        bk.p_lo = pmin < 0 ? 0 : pmin;
        bk.p_hi = pmax + 1 > S.P - 1 ? S.P - 1 : pmax + 1;
    }
    return bk;
}

// fill the work items of block `blk` once its position range is known (lanes split the channels).  A direct-target
// source's block has the reverberant items first, then as many direct items (direct spectra, `out_direct`): all of
// them carry the block's X, so k_render_fast stages it once for both stems.  Windowed source: only blocks that meet
// the window have items; output rows have stride win_len and sample n of the stem lands at row[n - win_start].  Every
// item carries `gain` (k_prepare passes stem_gain), direct items too: a direct stem takes its reverberant stem's gain.
SS_HD void fill_items(const Source& s, RItem* items, int blk, const Block& bk, int lane, int nlanes, float gain = 1.0f) {
    RItem it;
    it.X = s.xspec + (size_t)blk * kSpec;
    it.bounds = s.bounds; it.rstep = s.rstep; it.idx = s.idx; it.w = s.w;
    it.n0 = bk.start; it.n_end = bk.start + bk.len;
    it.n_lo = bk.start;
    const int ws = s.h_rows ? s.counts[4] : 0, wl = s.h_rows ? s.counts[5] : s.N;
    if (s.h_rows) {
        if (it.n_lo < ws) it.n_lo = ws;
        if (it.n_end > ws + wl) it.n_end = ws + wl;
    }
    it.mode = s.mode;
    const int reach = bk.start / kB + 1;
    it.kparts = reach < s.K ? reach : s.K;
    it.b0 = 0; it.step = 0.0; it.gain = gain;
    if (s.aligned) { it.b0 = s.bounds[bk.p_lo]; it.step = s.rstep[bk.p_lo]; }
    const int per = items_per_set(s);
    RItem* dst = items + s.counts[1] + (size_t)(blk - win_first(s)) * items_per_block(s);
    for (int i = lane; i < items_per_block(s); i += nlanes) {
        const bool direct = i >= per;
        const int c = direct ? i - per : i;
        // row r of the set at spec + (r - h_row0) * kSpec
        const float2* const spec = s.hspec + (direct ? (size_t)rows_stored_h(s) * kSpec : 0) - (ptrdiff_t)s.h_row0 * kSpec;
        float* const out = (direct ? s.out_direct : s.out) - ws;
        if (s.mode == MODE_STATIC) {                 // item c: channels 2c, 2c + 1
            it.H0 = spec + (size_t)(2 * c) * s.K * kSpec;
            it.row = out + (size_t)(2 * c) * wl;
            it.row1 = (2 * c + 1 < s.C) ? it.row + wl : nullptr;
            it.pstride = s.K * kSpec;
            it.p_lo = 0; it.p_hi = 0;
        } else {
            it.H0 = spec + (size_t)c * s.K * kSpec;
            it.row = out + (size_t)c * wl;
            it.row1 = nullptr;
            it.pstride = s.C * s.K * kSpec;
            it.p_lo = bk.p_lo; it.p_hi = bk.p_hi;
        }
        dst[i] = it;
    }
}

// The work items of a slot with a trajectory (take_trajectory), filled by k_blocks after its item scan (lane `lane` of
// `nlanes`): every block of the window as k_prepare's range warps fill it, then, for a reverse path, item position p
// moved to position P - 1 - p of the shifted set (H0 at the last visited position, the stride negated; the render
// kernels take H0 + (ptrdiff_t)p * pstride).  counts[0] = 0 afterwards (by the caller,
// once every lane is done) keeps k_prepare's range warps off the slot.
SS_HD void fill_traj_items(const Source& s, RItem* items, int lane, int nlanes) {
    const bool rev = (s.counts[25] & 2) != 0;
    const int first = win_first(s), per = items_per_block(s);
    for (int blk = first; blk < first + win_blocks(s); ++blk) {
        fill_items(s, items, blk, block_positions(s, s.blocks[blk], 0, 0), lane, nlanes, stem_gain(s));
        if (!rev) continue;
        RItem* const dst = items + s.counts[1] + (size_t)(blk - first) * per;
        for (int i = lane; i < per; i += nlanes) {         // the items this lane wrote
            dst[i].H0 += (ptrdiff_t)(s.P - 1) * dst[i].pstride;
            dst[i].pstride = -dst[i].pstride;
        }
    }
}

// k_render_fast: the two filter spectra of an item's single transform.  Aligned moving source: positions p_lo, p_lo + 1;
// static source: channels c, c + 1 - a static item without a partner channel reuses the first filter (its imaginary
// output is not stored).
SS_HD const float2* item_hp(const RItem& it) { return it.H0 + (ptrdiff_t)it.p_lo * it.pstride; }
SS_HD const float2* item_hq(const RItem& it) {
    const bool has = it.mode == MODE_STATIC ? it.row1 != nullptr : true;
    return item_hp(it) + (has ? it.pstride : 0);
}

// transform (item, p) -> descriptor
SS_HD XDesc make_xdesc(const RItem& it, int p) {
    XDesc d;
    d.X = it.X;
    d.Hp = it.H0 + (ptrdiff_t)p * it.pstride;
    const bool has_q = (it.mode == MODE_STATIC) ? (it.row1 != nullptr) : (p + 1 <= it.p_hi);
    d.Hq = has_q ? d.Hp + it.pstride : nullptr;
    d.row = it.row; d.row1 = it.row1;
    d.bounds = it.bounds; d.rstep = it.rstep; d.idx = it.idx; d.w = it.w;
    d.n0 = it.n0; d.n_end = it.n_end; d.p = p; d.p_lo = it.p_lo; d.p_hi = it.p_hi; d.n_lo = it.n_lo;
    d.first = (p == it.p_lo);
    d.valid = 1;
    d.mode = it.mode;
    d.kparts = it.kparts;
    d.gain = it.gain; d.pad_ = 0;
    return d;
}

// largest i with prefix[i] <= v, prefix[0] = 0, prefix has n+1 entries
SS_HD int find_source(const int* prefix, int n, int v) {
    int lo = 0, hi = n - 1;
    while (lo < hi) {
        int mid = (lo + hi + 1) >> 1;
        if (prefix[mid] <= v) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// =======================================================================================
// Spectra kernel: two real rows (a, b) -> one complex FFT -> two stored half spectra.
// A "row" is 8192 samples  a[n] = (0 <= g0 + n < len && n < ncap) ? base[g0 + n] : 0.
// =======================================================================================
struct Row {
    const float* src;      // base + g0: sample n of the row is src[n] for n in [nlo, nhi), zero elsewhere
    float2* dst;           // null -> row absent (odd count / unused block slot)
    int nlo, nspan;        // nspan = nhi - nlo (0: empty)
    float scale;
    float div;             // 0: samples as loaded; else every sample is divided by it first (SS_RIR_NORMALIZE)
};
SS_HD Row make_row(const float* base, float2* dst, int g0, int len, int ncap, float scale) {
    Row r;
    r.dst = dst; r.scale = scale; r.div = 0.f;
    int nlo = g0 < 0 ? -g0 : 0;
    int nhi = len - g0 < ncap ? len - g0 : ncap;
    r.nlo = nlo; r.nspan = nhi > nlo ? nhi - nlo : 0;
    r.src = base + g0;
    return r;
}
SS_HD Row no_row() { Row r; r.src = nullptr; r.dst = nullptr; r.nlo = 0; r.nspan = 0; r.scale = 0.f; r.div = 0.f; return r; }

// global abs-max of a normalised source's RIR tensor from k_rir_absmax's partial maxima
SS_HD float rir_absmax(const Source& s) {
    float m = 0.f;
    for (int i = 0; i < kNormParts; ++i) { const float v = s.norm_part[i]; m = v > m ? v : m; }
    return m;
}
// RIR row `row` (= (p * C + c) * K + partition) of set 0 (reverberant) or 1 (direct: the same taps, zero from
// cut[p, c] on - make_row zero-fills beyond `len`)
SS_HD Row make_row_h(const Source& s, int row, int set = 0) {
    if (row >= rows_h(s)) return no_row();
    int part = row % s.K, pc = row / s.K;
    const int len = set ? s.cut[pc] : s.L;
    Row r = make_row(s.rir + (size_t)pc * s.L, s.hspec + ((size_t)set * rows_stored_h(s) + (row - s.h_row0)) * kSpec,
                     part * kB, len, kB, 1.0f / (float)kF);
    if (s.norm_part) r.div = rir_absmax(s);
    return r;
}
// the two rows of k_prepare's RIR CTA `local` (< spectra_pairs_h): pairs of the reverberant set, then of the direct set
SS_HD void rows_of_pair_h(const Source& s, int local, Row& ra, Row& rb) {
    const int set = local >= pairs_per_set_h(s) ? 1 : 0, j = local - set * pairs_per_set_h(s);
    ra = make_row_h(s, s.h_row0 + 2 * j, set);
    rb = make_row_h(s, s.h_row0 + 2 * j + 1, set);
}
SS_HD Row make_row_x(const Source& s, int blk) {
    if (blk >= s.nblk_max) return no_row();
    const Block bk = s.blocks[blk];
    if (bk.len == 0) return no_row();
    return make_row(s.x, s.xspec + (size_t)blk * kSpec, bk.start - kB, s.N, kF, 1.0f);
}
SS_HD float row_at(const Row& r, int n) {
    return ((unsigned)(n - r.nlo) < (unsigned)r.nspan) ? r.src[n] : 0.f;
}
// IEEE single-precision division, what `ir_output /= ir_output.abs().max()` does per element (SonicSim_audio.py:398)
SS_HD float div_rn(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    return a / b;
#endif
}

// Direct-path cut of one RIR row (k_rir_direct; lane `lane` of `nlanes` scans taps lane, lane + nlanes, ...):
// first index of the maximum of |h| (|h / div| when div != 0, the bits k_prepare's row loads produce).  Partial
// results combine with peak_first, which prefers the smaller index on equal values, so the result is that of a
// sequential scan whatever the lane order.
struct PeakAt { float v; int i; };
SS_HD PeakAt peak_first(PeakAt a, PeakAt b) { return (b.v > a.v || (b.v == a.v && b.i < a.i)) ? b : a; }
SS_HD PeakAt peak_scan(const float* h, int L, float div, int lane, int nlanes) {
    PeakAt m; m.v = -1.f; m.i = 0;                   // below every |h|: an all-zero row peaks at 0
    for (int k = lane; k < L; k += nlanes) {
        const float a = fabsf(div != 0.f ? div_rn(h[k], div) : h[k]);
        if (a > m.v) { m.v = a; m.i = k; }
    }
    return m;
}
SS_HD int direct_cut(int peak, int L, int taps) { return peak < L - taps ? peak + taps : L; }   // min(L, peak + taps)

// ---- tap-form host banks (SS_BANK_TAPS, include/sonicsim_b200.h): a host bank that keeps each candidate's RIR taps as
// P*C*K rows of kB floats, row (p * C + c) * K + part holding taps [part * kB, part * kB + kB) of RIR (p, c), zero past
// L.  Tap j of row `row` as k_bank_taps stores it from bank_build's blockless source S (m: rir_absmax(S) of a normalised
// bank, else 0): divided as spectra_phase1 divides its row loads, never when m == 0, so that k_prepare over the stored
// rows without norm_part loads the values it loads over S with it - make_row's zero fill past L included (0 / m = +0).
SS_HD float tap_value(const Source& S, int row, int j, float m) {
    const int pc = row / S.K, t = (row % S.K) * kB + j;
    if (t >= S.L) return 0.f;
    const float h = S.rir[(size_t)pc * S.L + t];
    return m != 0.f ? div_rn(h, m) : h;
}
// The Source k_prepare's RIR CTAs transform a tap slot's staged rows [row0, row0 + rows) with: bank_build's blockless
// source over the stored rows (L = K * kB, so row r starts at rir + r * kB; rir biased: row r of the bank at
// staged + (r - row0) * kB), windowed onto the staged rows, which land in `spec` with set stride `rows` - the layout
// k_stage copies a spectral bank's rows into.  cut: the candidate's cut table for a slot with a direct stem, else null.
// `zero` is a zero word: CTAs past this run's spectra_pairs_h read counts[0] == 0 and return.
SS_HD Source tap_source(const float* staged, float2* spec, int* cut, int P, int C, int K, int row0, int rows,
                        int* zero) {
    Source s{};
    s.rir = staged - (ptrdiff_t)row0 * kB; s.N = 1; s.P = P; s.C = C; s.L = K * kB; s.K = K; s.nb = 1;
    s.mode = P == 1 ? MODE_STATIC : MODE_MOVING_BOUNDS;
    s.hspec = spec; s.cut = cut; s.counts = zero;
    s.h_row0 = row0; s.h_rows = rows;
    return s;
}
// What a slot of a tap-form pool stages besides its StageSlot (ss_kernels.cu), at the same index (k_stage<I16, true>):
struct StageTap {
    float* taps;                      // the staging area's tap rows (rows_cap * 4096 floats), or null: not a tap slot
    Source* src;                      // its transform Source (tap_source), written by CTA 0 at every run
    int* zero;                        // a zero word, the Source's counts
};
// A staged slot's area in a plan's descriptor allocation, every region at a 256-byte boundary from the area's start: its
// StageView, `sets` sets of rows_cap spectra rows, nx dry samples and, for a slot of a tap-form pool (taps), rows_cap
// rows of taps - the rows its transform turns into those spectra.  `end` is the area's size.
struct StageArea { size_t view, spec, x, taps, end; };
SS_HD size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }
SS_HD StageArea stage_area(int sets, int rows_cap, int nx, bool taps) {
    StageArea a;
    a.view = 0;
    a.spec = align256(sizeof(StageView));
    a.x = a.spec + align256((size_t)sets * rows_cap * kSpec * sizeof(float2));
    a.taps = a.x + align256(sizeof(float) * (size_t)nx);
    a.end = a.taps + (taps ? align256(sizeof(float) * (size_t)rows_cap * kB) : 0);
    return a;
}
// Behind a plan's staging areas, from the 256-aligned offset `at`, when it has slots of tap-form pools: one StageTap per
// staged slot, the n_tap transform Sources, their k_prepare CTA prefix (n_tap + 1 ints) and a zero word (the Sources'
// counts), each at a 256-byte boundary.  Offsets from the start of the allocation; `end` is where the block ends.
struct TapBlock { size_t taps, src, prefix, zero, end; };
SS_HD TapBlock tap_block(size_t at, int n_staged, int n_tap) {
    TapBlock t;
    t.taps = align256(at);
    t.src = t.taps + align256(sizeof(StageTap) * (size_t)n_staged);
    t.prefix = t.src + align256(sizeof(Source) * (size_t)n_tap);
    t.zero = t.prefix + align256(sizeof(int) * (size_t)(n_tap + 1));
    t.end = t.zero + 256;
    return t;
}

struct Regs32 { float2 a[16]; float2 b[16]; };

// S1: pass A of the forward transform straight from global memory: all 64 loads of the thread's two
// butterflies are issued before the first butterfly is computed (one exposed memory latency, not two).
SS_HD void spectra_phase1(int t, const Row& ra, const Row& rb, float2* s) {
    Regs32 R;
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        R.a[r] = make_float2(row_at(ra, t + 512 * r), row_at(rb, t + 512 * r));
        R.b[r] = make_float2(row_at(ra, t + 256 + 512 * r), row_at(rb, t + 256 + 512 * r));
    }
    if (ra.div != 0.f || rb.div != 0.f) {            // CTA-uniform: rows of a source whose RIRs are normalised on the fly
        const float da = ra.div != 0.f ? ra.div : 1.f, db = rb.div != 0.f ? rb.div : 1.f;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            R.a[r] = make_float2(div_rn(R.a[r].x, da), div_rn(R.a[r].y, db));
            R.b[r] = make_float2(div_rn(R.b[r].x, da), div_rn(R.b[r].y, db));
        }
    }
    fft16<false>(R.a); passA_store(s, t, R.a);
    fft16<false>(R.b); passA_store(s, t + 256, R.b);
}
// generic "load both butterflies t and t+256":  pad(t + 256) = pad(t) + 272
SS_HD void load2(int t, const float2* s, Regs32& R) {
    const float2* p = s + pad(t);
#pragma unroll
    for (int r = 0; r < 16; ++r) { R.a[r] = p[544 * r]; R.b[r] = p[544 * r + 272]; }
}

template <bool INV>
SS_HD void passB2(int t, float2* s, Regs32& R, const Tables& T) {
    passB_compute<INV>(t, R.a, T);       passB_store(s, t, R.a);
    passB_compute<INV>(t + 256, R.b, T); passB_store(s, t + 256, R.b);
}

// S3: pass C + closing radix-2, result (natural order) left in R: a[slot] = Zf[t + 256 r],
// b[slot] = Zf[4096 + t + 256 r], slot = out16(r).
SS_HD void spectra_phase3_compute(int t, Regs32& R, const Tables& T) {
    passC_compute<false>(t, R.a, T);
    passC_compute<false>(t + 256, R.b, T);
    float2 u[16];
    final_twiddles<false>(ldg_cached(T.tw + t), u);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        const int sl = out16(r);
        const float2 lo = R.a[sl], hi = cfma(lo, u[r], R.b[sl]);
        R.a[sl] = hi;
        R.b[sl] = twice_minus(lo, hi);
    }
}
// natural order to shared: pad(t + 256 r) = pad(t) + 272 r, pad(4096 + i) = 4352 + pad(i)
SS_HD void spectra_phase3_store(int t, float2* s, const Regs32& R) {
    float2* d = s + pad(t);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        d[272 * r] = R.a[out16(r)];
        d[272 * r + 4352] = R.b[out16(r)];
    }
}
// S4: split Zf into the spectra of a and b (Hermitian parts), scale, store.
SS_HD void spectra_phase4(int t, const float2* s, const Row& ra, const Row& rb) {
#pragma unroll 4
    for (int m = 0; m < 16; ++m) {
        int k = t + 256 * m;
        float2 A, Bv;
        if (k == 0) {
            float2 z0 = s[pad(0)], zn = s[pad(4096)];
            A = make_float2(z0.x, zn.x);
            Bv = make_float2(z0.y, zn.y);
        } else {
            float2 zk = s[pad(k)], zm = s[pad(kF - k)];
            A = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
            Bv = make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x));
        }
        if (ra.dst) ra.dst[k] = make_float2(A.x * ra.scale, A.y * ra.scale);
        if (rb.dst) rb.dst[k] = make_float2(Bv.x * rb.scale, Bv.y * rb.scale);
    }
}

// =======================================================================================
// Render kernel (inverse transform).  One CTA = one output block b of one channel (moving) or
// one channel pair (static).
// =======================================================================================

// RIR partitions >= 1 (long RIRs only), streamed from global memory and accumulated into the
// (P_A, P_B, Q_A, Q_B) slots of form_z.  Only instantiated in the LONG variant of k_render, which is
// launched for chunks that contain a source with L > 4096: keeping this loop (or even a call to it) out
// of the common kernel keeps the register allocation of its hot loop.
SS_HD void form_z_parts(int t, const XDesc& d, Regs32& R) {
    const int jB = passA_jB(t);
    const int kparts = d.kparts;
    const bool has_q = d.Hq != nullptr;
    for (int part = 1; part < kparts; ++part) {
        const float2* xa_p = d.X - (size_t)part * kSpec + t;
        const float2* xb_p = d.X - (size_t)part * kSpec + jB;
        const float2* ha_p = d.Hp + (size_t)part * kSpec + t;
        const float2* hb_p = d.Hp + (size_t)part * kSpec + jB;
        if (has_q) {
            const float2* ga_p = d.Hq + (size_t)part * kSpec + t;
            const float2* gb_p = d.Hq + (size_t)part * kSpec + jB;
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                float2 xa = ldg_stream(xa_p + 512 * m), xb = ldg_stream(xb_p + 512 * m);
                cmac(R.a[m], xa, ldg_stream(ha_p + 512 * m));
                cmac(R.b[m], xb, ldg_stream(hb_p + 512 * m));
                cmac(R.b[15 - m], xa, ldg_stream(ga_p + 512 * m));
                cmac(R.a[15 - m], xb, ldg_stream(gb_p + 512 * m));
            }
        } else {
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                float2 xa = ldg_stream(xa_p + 512 * m), xb = ldg_stream(xb_p + 512 * m);
                cmac(R.a[m], xa, ldg_stream(ha_p + 512 * m));
                cmac(R.b[m], xb, ldg_stream(hb_p + 512 * m));
            }
        }
    }
}

// Z formation fused with pass A.  sX / sHp / sHq: partition 0 of the dry window and of the two
// real filters packed into this transform, staged in shared memory (linear, 4096 words each) by the
// bulk-copy engine; sHq may be null.  RIR partitions j >= 1 (long RIRs) pair with the dry window
// 4096 j samples earlier (grid blocking) and are streamed from global memory through `d`.
template <bool LONG, bool FAST = false>
SS_HD void form_z(int t, const float2* sX, const float2* sHp, const float2* sHq, const XDesc& d, Regs32& R) {
    const int jB = passA_jB(t);
    {
        const float2 *xa_p = sX + t, *xb_p = sX + jB, *ha_p = sHp + t, *hb_p = sHp + jB;
        if (FAST || sHq) {          // FAST: every transform packs two positions (aligned blocking)
            const float2 *ga_p = sHq + t, *gb_p = sHq + jB;
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                float2 xa = xa_p[512 * m], xb = xb_p[512 * m];
                R.a[m] = cmul(xa, ha_p[512 * m]);            // P_A[m]
                R.b[m] = cmul(xb, hb_p[512 * m]);            // P_B[m]
                R.b[15 - m] = cmul(xa, ga_p[512 * m]);       // Q_A[m]
                R.a[15 - m] = cmul(xb, gb_p[512 * m]);       // Q_B[m]
            }
        } else {
#pragma unroll
            for (int m = 0; m < 8; ++m) {
                float2 xa = xa_p[512 * m], xb = xb_p[512 * m];
                R.a[m] = cmul(xa, ha_p[512 * m]);
                R.b[m] = cmul(xb, hb_p[512 * m]);
                R.b[15 - m] = make_float2(0.f, 0.f);
                R.a[15 - m] = make_float2(0.f, 0.f);
            }
        }
    }
    const int kparts = LONG ? d.kparts : 1;
    if (LONG) form_z_parts(t, d, R);
#pragma unroll
    for (int m = 0; m < 8; ++m) {
        float2 PA = R.a[m], QA = R.b[15 - m], PB = R.b[m], QB = R.a[15 - m];
        R.a[m] = z_direct(PA, QA);  R.b[15 - m] = z_mirror(PA, QA);
        R.b[m] = z_direct(PB, QB);  R.a[15 - m] = z_mirror(PB, QB);
    }
    if (t == 0) {
        // thread 0 owns the self-mirrored butterflies 0 and 256 and the packed (DC, Nyquist) word
        float2 x0 = sX[0], h0 = sHp[0];
        float pdc = x0.x * h0.x, pny = x0.y * h0.y, qdc = 0.f, qny = 0.f;
        if (FAST || sHq) { float2 g0 = sHq[0]; qdc = x0.x * g0.x; qny = x0.y * g0.y; }
        for (int part = 1; part < kparts; ++part) {
            x0 = (d.X - (size_t)part * kSpec)[0];
            h0 = (d.Hp + (size_t)part * kSpec)[0];
            pdc += x0.x * h0.x; pny += x0.y * h0.y;
            if (d.Hq) { float2 g0 = (d.Hq + (size_t)part * kSpec)[0]; qdc += x0.x * g0.x; qny += x0.y * g0.y; }
        }
        float2 tmp[8];
#pragma unroll
        for (int r = 8; r < 16; ++r) tmp[r - 8] = R.a[r];
#pragma unroll
        for (int r = 9; r < 16; ++r) R.a[r] = R.b[r - 1];
#pragma unroll
        for (int r = 8; r < 16; ++r) R.b[r] = tmp[r - 8];
        R.a[8] = make_float2(pny, qny);
        R.a[0] = make_float2(pdc, qdc);
    }
}
// ---- long RIRs (LONG): the partitions of a transform pass through the staging buffers one after the other.
// Stage j holds partition j of the two filters and the dry window 4096 j samples earlier (grid blocking);
// stage 0 initialises the product slots (P_A, P_B, Q_A, Q_B) of form_z, later stages accumulate, long_finish
// forms Z.  Thread 0 carries the packed (DC, Nyquist) products of all stages in `e`.
struct DcNy { float pdc, pny, qdc, qny; };
template <bool FIRST>
SS_HD void long_stage(int t, const float2* sX, const float2* sHp, const float2* sHq, Regs32& R, DcNy& e) {
    const int jB = passA_jB(t);
    const float2 *xa_p = sX + t, *xb_p = sX + jB, *ha_p = sHp + t, *hb_p = sHp + jB;
    if (sHq) {
        const float2 *ga_p = sHq + t, *gb_p = sHq + jB;
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const float2 xa = xa_p[512 * m], xb = xb_p[512 * m];
            if (FIRST) {
                R.a[m] = cmul(xa, ha_p[512 * m]);       R.b[m] = cmul(xb, hb_p[512 * m]);
                R.b[15 - m] = cmul(xa, ga_p[512 * m]);  R.a[15 - m] = cmul(xb, gb_p[512 * m]);
            } else {
                cmac(R.a[m], xa, ha_p[512 * m]);        cmac(R.b[m], xb, hb_p[512 * m]);
                cmac(R.b[15 - m], xa, ga_p[512 * m]);   cmac(R.a[15 - m], xb, gb_p[512 * m]);
            }
        }
    } else {
#pragma unroll
        for (int m = 0; m < 8; ++m) {
            const float2 xa = xa_p[512 * m], xb = xb_p[512 * m];
            if (FIRST) {
                R.a[m] = cmul(xa, ha_p[512 * m]);       R.b[m] = cmul(xb, hb_p[512 * m]);
                R.b[15 - m] = make_float2(0.f, 0.f);    R.a[15 - m] = make_float2(0.f, 0.f);
            } else {
                cmac(R.a[m], xa, ha_p[512 * m]);        cmac(R.b[m], xb, hb_p[512 * m]);
            }
        }
    }
    if (t == 0) {
        const float2 x0 = sX[0], h0 = sHp[0];
        if (FIRST) { e.pdc = x0.x * h0.x; e.pny = x0.y * h0.y; e.qdc = 0.f; e.qny = 0.f; }
        else { e.pdc += x0.x * h0.x; e.pny += x0.y * h0.y; }
        if (sHq) {
            const float2 g0 = sHq[0];
            if (FIRST) { e.qdc = x0.x * g0.x; e.qny = x0.y * g0.y; }
            else { e.qdc += x0.x * g0.x; e.qny += x0.y * g0.y; }
        }
    }
}
SS_HD void long_finish(int t, Regs32& R, const DcNy& e) {
#pragma unroll
    for (int m = 0; m < 8; ++m) {
        float2 PA = R.a[m], QA = R.b[15 - m], PB = R.b[m], QB = R.a[15 - m];
        R.a[m] = z_direct(PA, QA);  R.b[15 - m] = z_mirror(PA, QA);
        R.b[m] = z_direct(PB, QB);  R.a[15 - m] = z_mirror(PB, QB);
    }
    if (t == 0) {               // as in form_z: thread 0 owns butterflies 0 and 256 and the packed (DC, Nyquist) word
        float2 tmp[8];
#pragma unroll
        for (int r = 8; r < 16; ++r) tmp[r - 8] = R.a[r];
#pragma unroll
        for (int r = 9; r < 16; ++r) R.a[r] = R.b[r - 1];
#pragma unroll
        for (int r = 8; r < 16; ++r) R.b[r] = tmp[r - 8];
        R.a[8] = make_float2(e.pny, e.qny);
        R.a[0] = make_float2(e.pdc, e.qdc);
    }
}
SS_HD void render_phase1(int t, float2* s, Regs32& R) {
    fft16<true>(R.a); passA_store(s, passA_jA(t), R.a);
    fft16<true>(R.b); passA_store(s, passA_jB(t), R.b);
}

// pass C + closing radix-2 (second half only = the alias-free overlap-save samples):
// leaves z[4096 + t + 256 r] in R.a[out16(r)].
SS_HD void render_phase3(int t, Regs32& R, const Tables& T) {
    passC_compute<true>(t, R.a, T);
    passC_compute<true>(t + 256, R.b, T);
    float2 u[16];
    final_twiddles<true>(dirw<true>(ldg_cached(T.tw + t)), u);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        const int sl = out16(r);
        R.a[sl] = cfms(R.a[sl], u[r], R.b[sl]);
    }
}
// the closing radix-2 alone (pass C already done by the caller)
SS_HD void render_phase3_close(int t, Regs32& R, const Tables& T) {
    float2 u[16];
    final_twiddles<true>(dirw<true>(ldg_cached(T.tw + t)), u);
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        const int sl = out16(r);
        R.a[sl] = cfms(R.a[sl], u[r], R.b[sl]);
    }
}
// hat functions of positions (p, p+1) at a sample that lies in segment sg with weight w:
//   reference lerp (SonicSim_moving.py:94):  (1 - w) * conv[sg] + w * conv[sg + 1]
SS_HD void hat_pair(int sg, float w, int p, float& fa, float& fb) {
    const float omw = one_minus(w);
    fa = (sg == p) ? omw : ((sg + 1 == p) ? w : 0.f);
    fb = (sg == p + 1) ? omw : ((sg == p) ? w : 0.f);
}

// Output stage of one thread: samples n = n0 + t + 256 r, r = 0..15, visited in order.  `first` = first
// transform of its block (plain store); the second transform of a block that straddles a waypoint
// (grid blocking only) accumulates with a fire-and-forget RED - two addends per address, the first
// stored by this very thread, so the sum is order-free.  Every stored sample is v * gain (gain_mul).  Under a gain
// other than 1 a straddling block's first transform stores v unscaled and the last one (p + 2 > p_hi) replaces its RED
// by red_add_last, which scales the finished sum: the bits of accumulating first and scaling after (k_loud_scale).
template <bool FAST = false>
SS_HD void render_epilogue(int t, const XDesc& d, const Regs32& R) {
    // `d` lives in shared memory: copy what the loop needs into registers once - after every global
    // store the compiler would otherwise have to reload each field (generic pointers may alias)
    const int nbase = d.n0 + t, n_end = d.n_end, mode = d.mode, p = d.p;
    // samples stored: [n_lo, n_end), one unsigned compare (n_lo == n0 unless a window starts inside the block)
    const int n_lo = d.n_lo;
    const unsigned span = (unsigned)(n_end - n_lo);
    float* const row = d.row;
    const bool first = d.first != 0;
    const float g = d.gain;
    if (nbase >= n_end) return;
    if (!FAST && mode == MODE_STATIC) {                      // Re -> channel c, Im -> channel c + 1
        float* const row1 = d.row1;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int n = nbase + 256 * r;
            if ((unsigned)(n - n_lo) < span) {
                const float2 z = R.a[out16(r)];
                row[n] = gain_mul(z.x, g);
                if (row1) row1[n] = gain_mul(z.y, g);
            }
        }
    } else if (FAST || (mode == MODE_MOVING_BOUNDS && d.p_lo + 1 == d.p_hi)) {
        // the block lies inside one segment (always so under aligned blocking): sg = p for every
        // sample, 16 independent weight computations, lerp = (1 - w) Re z + w Im z
        // The 16 weights first, unguarded (no memory access), so that their int -> double -> float chains
        // interleave; (double)(n - b0) = d0 + 256 r exactly.
        const double d0 = (double)(nbase - d.bounds[p]);
        const double step = d.rstep[p];
        float w[16];
#pragma unroll
        for (int r = 0; r < 16; ++r) w[r] = (float)((d0 + 256.0 * r) * step);   // == np.linspace(0, 1, num, False)[i] as float32
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int n = nbase + 256 * r;
            const float2 z = R.a[out16(r)];
            const float v = gain_mul(lerp_terms(one_minus(w[r]), z.x, w[r], z.y), g);
            if ((unsigned)(n - n_lo) < span) row[n] = v;
        }
    } else if (mode == MODE_MOVING_BOUNDS) {
        const bool last = p + 2 > d.p_hi, fuse = last && g != 1.0f;
        const int* const bounds = d.bounds;
        const double* const rstep = d.rstep;
        int sg = d.p_lo;
        int b1 = bounds[sg + 1];
        while (nbase >= b1) { ++sg; b1 = bounds[sg + 1]; }
        int b0 = bounds[sg];
        double step = rstep[sg];
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int n = nbase + 256 * r;
            if ((unsigned)(n - n_lo) < span) {
                if (n >= b1) {
                    do { ++sg; b1 = bounds[sg + 1]; } while (n >= b1);
                    b0 = bounds[sg]; step = rstep[sg];
                }
                const float w = (float)((double)(n - b0) * step);
                float fa, fb;
                hat_pair(sg, w, p, fa, fb);
                const float2 z = R.a[out16(r)];
                const float v = lerp_terms(fa, z.x, fb, z.y);
                if (first) row[n] = last ? gain_mul(v, g) : v;
                else if (fuse) red_add_last(row + n, v, g);
                else red_add(row + n, v);
            }
        }
    } else {
        const bool last = p + 2 > d.p_hi, fuse = last && g != 1.0f;
        const int* const idx = d.idx;
        const float* const wv = d.w;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int n = nbase + 256 * r;
            if ((unsigned)(n - n_lo) < span) {
                float fa, fb;
                hat_pair(idx[n], wv[n], p, fa, fb);
                const float2 z = R.a[out16(r)];
                const float v = lerp_terms(fa, z.x, fb, z.y);
                if (first) row[n] = last ? gain_mul(v, g) : v;
                else if (fuse) red_add_last(row + n, v, g);
                else red_add(row + n, v);
            }
        }
    }
}

// Output stage of k_render_fast (aligned blocking: the block lies in segment p_lo, one transform per item): as the
// single-segment branch above, with the segment's first sample and 1 / length taken from the work item itself.
// GAIN = false (chunks without a pooled slot of a pool with gains, where every item's gain is 1) stores without the
// multiply, which costs the issue-bound kernel about 2 %.
template <bool GAIN = true>
SS_HD void render_epilogue_item(int t, const RItem& it, const Regs32& R) {
    const int nbase = it.n0 + t, n_end = it.n_end;
    const int n_lo = it.n_lo;                                // stored: [n_lo, n_end), as in render_epilogue
    const unsigned span = (unsigned)(n_end - n_lo);
    float* const row = it.row;
    const float g = it.gain;
    if (nbase >= n_end) return;
    if (it.mode == MODE_STATIC) {                            // Re -> channel c, Im -> channel c + 1 (item-uniform branch)
        float* const row1 = it.row1;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int n = nbase + 256 * r;
            if ((unsigned)(n - n_lo) < span) {
                const float2 z = R.a[out16(r)];
                row[n] = GAIN ? gain_mul(z.x, g) : z.x;
                if (row1) row1[n] = GAIN ? gain_mul(z.y, g) : z.y;
            }
        }
        return;
    }
    const double d0 = (double)(nbase - it.b0);
    const double step = it.step;
    float w[16];
#pragma unroll
    for (int r = 0; r < 16; ++r) w[r] = (float)((d0 + 256.0 * r) * step);   // == np.linspace(0, 1, num, False)[i] as float32
#pragma unroll
    for (int r = 0; r < 16; ++r) {
        const int n = nbase + 256 * r;
        const float v = GAIN ? gain_mul(lerp_pair(w[r], R.a[out16(r)]), g) : lerp_pair(w[r], R.a[out16(r)]);
        if ((unsigned)(n - n_lo) < span) row[n] = v;
    }
}

}  // namespace ss
