/* sonicsim_b200.h - C ABI of the H100-native moving-source renderer.
 *
 * The reference (JusperLee/SonicSim) has no FFI layer: its hot path is module-level Python
 * (SonicSim-SonicSet/SonicSim_moving.py, SonicSim_audio.py) called positionally from
 * SonicSet.py:77-101.  This header is the native boundary a maintainer binds instead (ctypes stub
 * in INTEGRATION.md; sonicsim_b200/_lib.py is that stub).  Each entry point names the reference
 * function(s) it replaces.  Plain pointers and sizes only; no torch / Python types.
 *
 * Conventions
 *   - float32 everywhere, row-major.  dry x: (N,), RIRs: (P, C, L), output: (C, N) channel-major.
 *   - `*_dev` entry points take DEVICE pointers and enqueue work on `stream` (a cudaStream_t cast to
 *     void*; NULL = legacy default stream) without synchronising.
 *   - `*_host` entry points take HOST pointers (pinned memory gives full PCIe rate), copy in,
 *     render and copy out; they return after the results are in host memory.
 *   - an ss_ctx is NOT thread-safe: use one context per host thread (one process per GPU is the
 *     intended deployment); calls on one context are serialised by the caller.
 *   - streams: a call on one stream may follow a call on another (or a host call) at once.  The library orders its
 *     own buffers - scratch, descriptor blocks, a bank or pool under construction - behind their earlier users on
 *     every stream, on the device (only a descriptor block's pinned staging copy, reused every 6 calls or chunks, may
 *     hold the host until its previous upload is done).  The caller orders only its own buffers: an input written or an output
 *     read on another stream needs the caller's event or synchronisation, as for any CUDA work.  Two runs of one plan
 *     write the same outputs, so they are the caller's to order.
 *   - every function returns 0 (SS_OK) or a negative ss_status; ss_strerror() describes it.  The
 *     Python shim turns these into the exception types the reference raises (IndexError /
 *     ValueError), see INTEGRATION.md.
 */
#ifndef SONICSIM_B200_H_
#define SONICSIM_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ss_ctx ss_ctx;
typedef struct ss_bank ss_bank;
typedef struct ss_pool ss_pool;
typedef struct ss_dry_pool ss_dry_pool;
typedef struct ss_pair_gains ss_pair_gains;

typedef enum {
    SS_OK = 0,
    SS_ERR_INVALID = -1,      /* bad argument (null pointer, non-positive size, unknown mode)       */
    SS_ERR_INDEX = -2,        /* trajectory refers to a position >= P - 1 (reference: IndexError)   */
    SS_ERR_CUDA = -3,         /* CUDA runtime error; ss_last_cuda_error() has the code              */
    SS_ERR_NOMEM = -4,        /* device or pinned allocation failed                                 */
    SS_ERR_UNSUPPORTED = -5   /* shape outside what this build handles                              */
} ss_status;

/* how one source's trajectory is given */
typedef enum {
    SS_STATIC = 0,            /* P == 1, no interpolation: convolve_fixed_receiver                  */
    SS_MOVING_BOUNDS = 1,     /* `bounds`: P int32 cumulative segment bounds, bounds[0]=0, [P-1]=N   */
    SS_MOVING_INDEXED = 2     /* `idx` (int32, N) and `w` (float32, N): interp_index / interp_weight */
} ss_mode;

/* per-source options (ss_source.flags) */
typedef enum {
    SS_RIR_NORMALIZE = 1,     /* `rir` is the raw simulator output, clipped and stacked: divide every tap by the global
                               * abs-max of the source's whole (P, C, L) tensor before convolving, i.e. the
                               * `ir_output /= ir_output.abs().max()` of generate_rir_combination
                               * (SonicSim_audio.py:391-398), fused into the spectra kernel's row loads (one reduction
                               * kernel + an IEEE division per tap; same bits as normalising first) */
    SS_DIRECT_TARGET = 2      /* also render the direct-path stem into `out_direct` (speech-enhancement /
                               * dereverberation target), in the same launches as the reverberant stem `out`.
                               * Each row h[p, c, :] (after normalisation when SS_RIR_NORMALIZE is set) is cut after
                               *   peak[p, c] = first index of max_k |h[p, c, k]|   (np.argmax's tie rule; 0 for an
                               *                                                     all-zero row)
                               *   cut[p, c]  = min(L, peak[p, c] + direct_taps)
                               * i.e. h_d[p, c, k] = h[p, c, k] for k < cut[p, c], 0 otherwise, and rendered with the
                               * source's own trajectory, blocking and weights: `out_direct` has the bits of rendering h_d
                               * as a separate source of the same mode, `out` the bits of the source without this flag.
                               * The peak is the strongest tap, which in a simulated RIR may be a reflection rather
                               * than the earliest arrival.  direct_taps = 40 is 2.5 ms at 16 kHz; a longer one (e.g.
                               * 50 ms) gives an early-reflections target.  With ss_render_host_ex loudness
                               * normalisation the direct stem is scaled by the reverberant stem's gain. */
} ss_source_flags;

/* One (utterance, source) unit of work = one call of convolve_moving_receiver /
 * convolve_fixed_receiver in the reference.  Pointers are device pointers for ss_render_dev and
 * host pointers for ss_render_host. */
typedef struct {
    const float* x;           /* (N,)       dry source, SonicSim_moving.py:64                        */
    const float* rir;         /* (P, C, L)  per-position RIRs, SonicSim_moving.py:65; (C, L) if static;
                               *            NULL with `rir_bank`                                        */
    float* out;               /* (C, N)     rendered stem, SonicSim_moving.py:96 / :60               */
    const int32_t* bounds;    /* SS_MOVING_BOUNDS: np.cumsum(samples_per_interval) with leading 0    */
    const int32_t* idx;       /* SS_MOVING_INDEXED: interp_index (SonicSim_moving.py:42)             */
    const float* w;           /* SS_MOVING_INDEXED: interp_weight (SonicSim_moving.py:43)            */
    int32_t N, P, C, L;
    int32_t mode;             /* ss_mode */
    int32_t flags;            /* ss_source_flags, 0 = none */
    const int32_t* bounds_host; /* ss_render_dev only, optional: HOST copy of `bounds` (P ints).  With it the block
                                 * table is built on the host and one small kernel launch per chunk is saved.     */
    float* out_direct;        /* SS_DIRECT_TARGET: (C, N) direct-path stem, same pointer kind as `out`, != out    */
    int32_t direct_taps;      /* SS_DIRECT_TARGET: taps kept from each row's peak on, >= 1                        */
    int32_t win_start, win_len; /* time window, see below; win_len == 0: the whole stem                          */
    const ss_bank* rir_bank;  /* RIR spectrum bank (version 103) instead of `rir`, which is then NULL; see below   */
    const int32_t* win_start_dev; /* moving window (version 104): DEVICE pointer to the start, read at every run in
                                   * place of win_start; see below                                                  */
    const ss_pool* pool;      /* pooled slot (version 106): the source rendered is the candidate of `pool` ...      */
    const int32_t* pick_dev;  /* ... named by the int32 at this DEVICE pointer, read at every run; see below         */
} ss_source;                  /* fields appended since version 100: a zeroed (memset) struct leaves them off      */

/* Time window (win_len > 0, version 102): the source renders only output samples [win_start, win_start + win_len)
 * with 0 <= win_start and win_start + win_len <= N.  `out` (and `out_direct`) is then a dense (C, win_len) buffer,
 * row stride win_len, and every value stored has the bits of the same sample of the full render of the same source by
 * the same kernel variant: the blocking is chosen over the whole trajectory and length N exactly as for the full stem
 * (ss_debug_plan), and only the blocks that meet the window are rendered.  The kernel variant depends on the source's
 * kind - one transform per block (aligned blocking, or static with L <= 4096), L > 4096, or any other - and never on
 * its window.  ss_render_dev and plans run each kind on its own variant, so there a window always has the bits of the
 * full stem.  ss_render_host renders each of its chunks with one variant: a chunk that mixes kinds takes the most
 * general one present, whose roundings may differ from those of the one-transform kernel.  A host-path window therefore
 * has the full stem's bits when both are rendered in batches whose sources are all of its kind.  Whole stems on the
 * host path depend on their batch in the same way.  A loudness target of ss_render_host_ex cannot be combined with a
 * window (the reference normalises the whole stem; a window does not know that stem's gain): SS_ERR_INVALID.
 *
 * Read set of a windowed source - everything outside it may hold anything (NaN, garbage; on the host path it is not
 * even copied):
 *   - dry x: the windows [start - 4096, start + 4096) of the blocks that meet the window, of the RIR partitions'
 *     K - 1 = ceil(L / 4096) - 1 grid blocks in front of the first of them, and of the partner block each of these
 *     is paired with in the forward transform (blocks 2i and 2i + 1 of the full plan share one FFT);
 *   - bounds: all P entries;  idx / w (SS_MOVING_INDEXED): the samples of the blocks that meet the window;
 *   - RIR positions: every position a block that meets the window interpolates between, widened to the rows paired
 *     with them in the forward transform (rows 2r and 2r + 1 of the P * C * K row list share one FFT: when C * K is
 *     odd, the last row of the position in front may be read);  all P positions under SS_RIR_NORMALIZE (the global
 *     abs-max) and whenever the trajectory is not visible on the host (SS_MOVING_INDEXED, or a device `bounds` without
 *     `bounds_host`).
 * A source with a `rir_bank` reads no RIR positions at all, windowed or not.
 * On the device path, ss_device_errors reports only what the kernels read: the idx entries of the read set, and the
 * bounds table of a grid-blocked source.
 *
 * Moving window (version 104): `win_start_dev` points to one int32 in device memory (4-byte aligned) that holds the
 * start, so that a crop can move between runs of a plan (or be drawn on the device) without any host work.  Only with
 * win_len > 0 and win_start == 0; anything else, or an unaligned pointer, is SS_ERR_INVALID before any work.
 * ss_render_dev and ss_plan_create take such sources; ss_render_host / _ex refuse them (SS_ERR_INVALID): the host path
 * copies a read set that depends on the start.  The value is read when the run's first kernel reaches it: write it on
 * the run's stream, or in an order that is guaranteed to come before that stream.  A start outside [0, N - win_len] is
 * clamped into that range, the window is rendered there, and ss_device_errors reports bit 2.  win_len fixes the output
 * shape and stays bound.  Bits, blocking and kernel variant are those of a fixed window at the same start.  A chunk that
 * holds a moving window builds its block tables on the device (k_blocks, as without bounds_host), sized once for the
 * largest table any start needs.  Read set: all of x; all of bounds / idx / w; all P RIR positions (the RIR rows of
 * every position are transformed at every run), none with a `rir_bank` - a bank is the way to crop a fixed RIR set
 * step after step without transforming it again. */

/* ---- RIR spectrum banks (version 103).  The half spectra of a source's RIR partitions depend on nothing but its taps,
 * SS_RIR_NORMALIZE and direct_taps - not on the dry signal, the trajectory, the window or the batch.  A bank holds them
 * in device memory, transformed once by the same kernels and in the same layout as every render transforms them into
 * its scratch: (P, C, K = ceil(L / 4096), 4096) complex64 pre-scaled by 1/8192, with a direct set a second block of
 * that shape right behind it and the P * C cut table.  A source that names a bank renders bit-identically to the same
 * source given the raw RIRs (same flags, through the same kernel variant), without transforming, copying or reading
 * any RIR: re-rendering a fixed RIR set (a trajectory of an RIR dump, a training scene) with new dry signals.
 *
 * rir: (P, C, L) float32, or (C, L) with P = 1 for a static source.  flags: SS_RIR_NORMALIZE (the bank holds the
 * normalised taps' spectra) and / or SS_DIRECT_TARGET (also the direct-path set, direct_taps >= 1; see that flag).
 * _dev: device pointer, asynchronous on `stream`: the caller keeps `rir` unchanged until the stream gets there.  The bank
 * records an event behind its construction, and every call that uses it - ss_render_dev (on its `stream`),
 * ss_render_host / _ex (on the context's own streams) and every ss_plan_run - makes its work wait on that event, so a
 * render never reads a bank that is still being built, whatever stream built it.  _host: host pointer, returns when the
 * bank is complete.  The bank holds 8 * 4096 * P * C * K bytes per set (ss_bank_bytes: everything it holds on the device).
 *
 * A source that uses a bank (every violation is SS_ERR_INVALID, before any work):
 *   - sets `rir_bank` and leaves `rir` NULL;
 *   - has the bank's P, C and L; a static source takes a bank with P == 1, a moving source one with P >= 2;
 *   - does not set SS_RIR_NORMALIZE (normalisation is a property of the bank);
 *   - sets SS_DIRECT_TARGET only with a bank that holds a direct set, and then with the bank's direct_taps (a bank with
 *     a direct set also serves sources that render only the reverberant stem);
 *   - is rendered with the context that created the bank (and so on its device).
 * Windows, ss_render_host_ex loudness targets and plans work with banked sources as with raw RIRs.  Lifetime: a bank
 * must outlive every call and every plan that uses it (see the plan rules below); ss_bank_destroy waits for the device
 * before it frees the bank, like ss_plan_destroy.  Bank bytes are not part of the chunk budget (ss_set_chunk_bytes). */
int ss_bank_create_dev(ss_ctx* ctx, const float* rir, int32_t P, int32_t C, int32_t L, int32_t flags,
                       int32_t direct_taps, void* stream, ss_bank** out);
int ss_bank_create_host(ss_ctx* ctx, const float* rir, int32_t P, int32_t C, int32_t L, int32_t flags,
                        int32_t direct_taps, ss_bank** out);
int64_t ss_bank_bytes(const ss_bank* bank);   /* device bytes held */
void ss_bank_destroy(ss_bank* bank);          /* destroy banks before their context */

/* ---- host banks: `flags` of ss_bank_create_dev / _host may add SS_BANK_HOST.  The bank is transformed by the same
 * launches into a transient device buffer, then moved into pinned, mapped host memory (cudaHostAllocMapped) - spectra and
 * cut table alike - and the device buffer is freed: its spectra are bit-identical to a device bank's of the same RIRs,
 * ss_bank_bytes is 0 and ss_bank_host_bytes reports the 8 * 4096 * P * C * K bytes per set plus the cut table.  Both
 * create calls return only when the bank is in host memory.  A host bank serves only as a candidate of a host pool
 * (below): ss_render_dev, ss_render_host / _ex and ss_plan_create* refuse a source that names one (SS_ERR_INVALID). */
#define SS_BANK_HOST 0x100
int64_t ss_bank_host_bytes(const ss_bank* bank);   /* pinned host bytes held */

/* ---- tap-form host banks: `flags` may add SS_BANK_TAPS together with SS_BANK_HOST (without it the create calls return
 * SS_ERR_INVALID before any allocation); it combines with SS_RIR_NORMALIZE and SS_DIRECT_TARGET as the spectral form
 * does.  Such a bank keeps the taps instead of their spectra: pinned, mapped host memory holds P * C * K rows of 4096
 * float32, row (p * C + c) * K + part at float offset row * 4096 holding taps [part * 4096, part * 4096 + 4096) of RIR
 * (p, c), zero past L, then the cut table as in a spectral host bank.  With SS_RIR_NORMALIZE the stored taps are the
 * IEEE quotients h / m, m the abs-max of the whole RIR tensor (k_rir_absmax), and the raw taps when m == 0.  The build runs
 * k_rir_absmax and k_rir_direct as for a spectral bank, then writes the rows; nothing is transformed.
 * ss_bank_host_bytes = 16384 * P * C * K plus 4 * P * C with a direct set (half a spectral host bank's bytes, a quarter
 * with a direct set); ss_bank_bytes is 0.  A tap-form bank serves only as a candidate of a host pool whose banks are all
 * tap-form (a pool that mixes forms is SS_ERR_INVALID).  Such a pool stages, at every run, the rows [row0, row0 + rows)
 * of its slots' read sets as rows * 16 KB - one set whatever the slot's direct target - instead of sets * rows * 32 KB of
 * spectra, and one more kernel per run, a k_prepare launch behind k_stage and before any chunk, transforms them on the
 * device into the staging area's spectra, rows paired (2r, 2r + 1) as a bank build pairs them.
 * Bit contract: a plan over tap-form host pools gives the bits of the same plan over spectral host pools of the same RIRs
 * - and so of device pools - in stems, direct stems, mixtures, speakers_out, rms_db, drawn starts, `used` and
 * ss_device_errors, for dry picks and pair gains too; level tables, loudness results and pair gains are identical.  The
 * transform loads the values a spectral build loads (pre-divided taps, zeros past L for its zero fill, direct rows cut at
 * the same cut[p, c]), through the same code.  ss_version stays 108: ss_bank_flags marks the capability. */
#define SS_BANK_TAPS 0x200
int32_t ss_bank_flags(const ss_bank* bank);        /* the flags the bank was created with (0 for NULL) */

/* ---- source pools (version 106): the dataloader's random choices of separation/look2hear/datas/movingdatamodule.py
 * :57-59 (`random.choice(self.data_dirs)`, `random.sample(range(1, 4), num_spks)`) and :68-77 (the scene's noise) made
 * on the device.  A pool is a set of banked candidate sources, validated and uploaded once.  A pooled slot of a plan
 * (ss_source.pool + pick_dev) renders, at every run, the candidate named by the int32 at pick_dev: its dry signal,
 * trajectory, N, P and bank.  The slot's outputs, window length, flags and mixture membership stay bound.  Bits, blocking
 * and kernel variant are those of the picked candidate rendered as a windowed source at the same (clamped) start under
 * the pool's blocking (below); when every candidate would choose that blocking on its own, a pooled output equals
 * ss_render_dev of the picked candidate with the same window, bit for bit.
 *
 * Candidates (every violation is SS_ERR_INVALID, before anything is allocated):
 *   - 1 <= n <= 2^24;
 *   - banked: rir == NULL, rir_bank set, a bank of this context, with the candidate's P, C and L; `x` set;
 *   - one `mode` for all, SS_MOVING_BOUNDS or SS_STATIC (SS_MOVING_INDEXED is refused), one C; L may differ
 *     (SonicSet gives every speaker of a scene its own RIR length): each candidate keeps its own bank, unpadded;
 *   - a moving candidate has `bounds` and `bounds_host` (ascending from 0 to N), so that the pool's blocking and table
 *     sizes are exact; idx and w are NULL;
 *   - out, out_direct, flags, direct_taps, win_start, win_len, win_start_dev, pool and pick_dev are zero.
 * Banks with and without a direct set may be mixed in one pool; the direct rule is enforced per slot.
 * Blocking: aligned if every candidate would choose aligned blocking on its own (ss_debug_plan) with its own
 * K = ceil(L / 4096), otherwise the 4096-sample grid for all of them.  The kernel variant of a pooled slot is fixed when
 * the pool is created, from the pool's largest K: k_render<LONG> if any candidate has K > 1.  A slot that picks candidate
 * i renders with that candidate's own K_i RIR partitions.  A pool's L is its longest candidate's.
 * Bits of candidates of different L: a candidate that would choose the pool's blocking and variant on its own (every
 * K_i > 1 candidate, and every candidate of a pool whose candidates share K) has the bits of ss_render_dev as above.  A
 * K_i = 1 candidate of a pool with K > 1 candidates runs k_render<LONG> with one partition: its output equals, bit for
 * bit, a render over its bank with exact-zero partitions appended, and the render of its RIRs zero-padded to the pool's
 * L within float32 rounding only (a padded bank's zero partitions hold the rounding residue of the rows they are
 * transformed with).  Level tables and gains (below) are computed from every candidate rendered whole on its own, so
 * for such a candidate they differ from its pooled stems by float32 rounding, as for a candidate that chooses other
 * blocking than its pool.
 * The pool copies what it needs (including the bounds_host values); the candidates' device buffers (x, bounds) and banks
 * must outlive the pool.  ss_pool_create returns when the pool's table is in device memory; the pool records one event
 * behind the construction of all its banks, which every plan run that uses the pool waits on.
 *
 * A pooled slot (every violation is SS_ERR_INVALID, before anything is allocated):
 *   - x, rir, rir_bank, bounds, bounds_host, idx and w are NULL, N and P are 0; pool of this context; pick_dev a 4-byte
 *     aligned device pointer;
 *   - mode, C and L are the pool's (L: the longest candidate's);
 *   - win_len > 0 with a fixed win_start (win_start + win_len <= every candidate's N) or a win_start_dev (win_start == 0
 *     and win_len <= every candidate's N); the window start is clamped against the picked candidate's N (bit 2);
 *   - SS_DIRECT_TARGET only if every candidate's bank holds a direct set with the slot's direct_taps; no
 *     SS_RIR_NORMALIZE (normalisation is a property of the banks).
 * ss_plan_create and ss_plan_create_mix take pooled slots; ss_render_dev, ss_render_host and ss_render_host_ex refuse
 * them (SS_ERR_INVALID).  The pick is read when the run's first kernel reaches it (as win_start_dev); a pick outside
 * [0, n) is clamped into that range and ss_device_errors reports bit 3.  Read set of a pooled slot: the picked
 * candidate's whole x and bounds (and its bank); for the mixture range checks of ss_plan_create_mix, every candidate's x
 * and bounds and the pick.  A chunk that holds a pooled slot builds its block tables on the device, sized once, when the
 * plan is created, for the largest any candidate needs: 3 kernel launches per chunk, as with a moving window.
 * Lifetime: a pool must outlive every plan that uses it; ss_pool_destroy waits for the device before it frees it. */
int ss_pool_create(ss_ctx* ctx, const ss_source* candidates, int n, ss_pool** out);
int64_t ss_pool_bytes(const ss_pool* pool);   /* device bytes held: n compact candidate entries (40 B each), the n
                                               * int32 partition counts (4 B each) when the candidates' K differ, the n
                                               * float gains (4 B each) once ss_pool_loudness measured them, and the
                                               * level tables with their pointer array once ss_pool_levels built them */
void ss_pool_destroy(ss_pool* pool);          /* destroy pools after the plans that use them, before their context */

/* ---- host pools: a pool whose candidates all have host banks (SS_BANK_HOST) is a host pool; a pool that mixes host and
 * device banks is SS_ERR_INVALID.  Its bulk stays in pinned host memory and every plan run copies only what its slots
 * read into device memory, so that a pool's device footprint is O(n * P) bytes whatever its dry signals and banks hold.
 *   - ss_pool_create copies every candidate's `x` (a host or a device pointer) into one pinned, mapped arena that the pool
 *     owns, uploads each moving candidate's bounds_host into a device array of its own (`bounds` may then be NULL), and
 *     uploads the direct-path cut tables (P * C ints per candidate whose bank has a direct set).  Unlike a device pool,
 *     the caller's x and bounds buffers need not outlive the pool: only the banks must.
 *   - ss_pool_levels puts the tables in pinned, mapped host memory (ss_pool_level_table then returns a mapped host
 *     address, which the device reads over PCIe); ss_pool_levels and ss_pool_loudness render each stem group from
 *     transient device copies of its banks and dry signals, in batches of at most 256 MB (or one candidate's, when
 *     larger), so that a build's transient device memory is bounded whatever n is.
 *   - In a plan, every pooled slot of a host pool gets a staging area in device memory, sized once at creation for the
 *     most RIR rows (both sets with a direct target) and dry samples any candidate's window of this length reads at any
 *     start.  At every run one more kernel, k_stage, launched after the start draws and before any render, reads each
 *     such slot's pick (clamped, bit 3) and start, and copies the picked candidate's read set from host memory into the
 *     staging area: the dry samples [ws - (K + 2) * 4096, ws + win_len + 2 * 4096) and the RIR rows of every position
 *     they reach.  The slot then renders from the staged copies with the bits of the same slot over a device pool.
 *   - ss_pool_bytes keeps counting device bytes: for a host pool the n entries, the partition counts and gains as for a
 *     device pool, the device copies of the bounds (4 * P bytes per moving candidate) and cut tables, and the level
 *     tables' pointer array; ss_pool_host_bytes counts the arena and the level tables.
 *   - Dry picks (ss_dry_pick, below) on a host pool's slots take a host dry pool (SS_DRY_HOST): k_stage then copies the
 *     same dry samples from the picked dry signal instead of the candidate's x.  A device dry pool is refused there. */
int64_t ss_pool_host_bytes(const ss_pool* pool);   /* pinned host bytes held (0 for a device pool) */

/* ---- level tables of a pool (version 107), for the start draws of plans (ss_plan_draw below).  Gives every candidate
 * of the pool a table from which the energy of any crop is two loads:
 *   Q[0] = 0, Q[n + 1] = Q[n] + e[n] for n < N, in float64 (N + 1 doubles), where e[n] is computed from the candidate's
 *   whole reverberant stem as ss_render_dev renders it (the candidate as a whole banked source, bounds_host included),
 *   the normalised stem - that stem times (float)gain, with k_loud_scale's arithmetic - in a pool with gains
 *   (ss_pool_loudness below):
 *     - flags = SS_MIX_MONO: e[n] = (double)(v * v), v the channel fold of the mixture kernels at n (SS_MIX_MONO of
 *       ss_plan_mix: the float32 sum of the C rows in channel order, then an IEEE division by C), with the same bits;
 *     - flags = 0: e[n] = sum over c of (double)(y[c, n] * y[c, n]), in channel order.
 *   These are the terms a mixture's rms_db sums, so a crop's level from a table differs from the plan's rms_db of the
 *   same crop only by the order of the float64 sums.  The scan has a fixed order: identical bits at every build.
 * The candidates are rendered in groups through the device path into one transient buffer of at most 256 MB (or one
 * candidate's stem, when larger), after the pool's banks are complete.  Returns when the tables are in device memory.
 * The tables cost 8 bytes per sample (3.84 MB for a 30 s candidate at 16 kHz) and describe the candidates' dry signals
 * as they are at this call: a pool whose `x` buffers change afterwards needs a new pool for new tables.
 * Refused (SS_ERR_INVALID): a NULL pool, flags other than 0 / SS_MIX_MONO, a pool that already has tables. */
int ss_pool_levels(ss_pool* pool, uint32_t flags);
/* Device pointer of candidate i's table (N + 1 doubles), or NULL without tables or with i outside [0, n). */
const double* ss_pool_level_table(const ss_pool* pool, int i);

/* library / build identification */
int ss_version(void);        /* 108: loudness gains of pools (ss_pool_loudness) */
const char* ss_strerror(int status);
int ss_last_cuda_error(void);

/* One context per process per GPU: owns the twiddle table, scratch for spectra and the staging
 * buffers / streams of the host path.  `device` is the CUDA ordinal (after CUDA_VISIBLE_DEVICES). */
int ss_create(int device, ss_ctx** out);
void ss_destroy(ss_ctx* ctx);

/* Tunables: scratch budget per launch group (bytes of spectra kept live, sized to stay in L2). */
int ss_set_chunk_bytes(ss_ctx* ctx, int64_t bytes);

/* Replaces SonicSim_moving.convolve_moving_receiver (SonicSim_moving.py:63-96) and
 * convolve_fixed_receiver (:47-61) for a whole batch of sources in two (three without bounds_host) kernel
 * launches per chunk.  Device pointers; asynchronous on `stream`.
 * Preconditions the device path cannot check without a round trip (the host path checks them and returns
 * SS_ERR_INDEX / SS_ERR_INVALID like the reference raises): SS_MOVING_INDEXED: 0 <= idx[n] <= P - 2 for every n
 * (out-of-range samples are rendered as zeros, not reported); SS_MOVING_BOUNDS without bounds_host: bounds is
 * non-decreasing with bounds[0] = 0 and bounds[P - 1] = N (anything else is undefined behaviour). */
int ss_render_dev(ss_ctx* ctx, const ss_source* items, int n_items, void* stream);

/* The device path cannot return SS_ERR_INDEX: kernels that meet a trajectory outside the contract above render the
 * offending samples as silence (clamped positions) and set a bit that this call returns and clears after waiting for
 * the device: bit 0 = an interp_index outside [0, P - 2], bit 1 = a device-side bounds table that is not ascending from
 * 0 to N (checked for grid-blocked sources), bit 2 (version 104) = a moving window's start outside [0, N - win_len]
 * (rendered clamped into that range), bit 3 (version 106) = a pooled slot's pick outside [0, n) (clamped), bit 4 (dry
 * pools, below) = a dry pick outside [0, n) of its dry pool (clamped), bit 5 (dry streams and background streams,
 * below) = an invalid entry of a stream or bed slot's layout (skipped), bit 6 (loudness slots, ss_stream_lufs below) =
 * a loudness target read at a run that was not finite (that slot stored unscaled), bit 7 (speaker groups,
 * ss_layout_group below) = a grouped layout draw's group outside [0, G) (clamped), bit 8 (trajectories, ss_trajectory
 * below) = an invalid path or bounds table of a pooled slot (its candidate's own path rendered).  The Python device API raises
 * IndexError / ValueError from it on request
 * (Renderer.check_device_errors).  The bits live in one device word per GPU, shared by every context of the
 * process on that GPU: with several such contexts, a call on one returns and clears the bits another one's kernels set. */
int ss_device_errors(ss_ctx* ctx, uint32_t* bits);

/* A batch of device-resident sources bound once (the generation loop of SonicSet.py:180-214 renders the same
 * shapes scene after scene into the same buffers).  ss_plan_create validates, chunks, builds the block tables and
 * keeps the descriptor blocks and the scratch for the spectra resident; ss_plan_run is then kernel launches only,
 * issued as ONE CUDA graph launch on `stream` (captured on the first run; the launches fork over the context's
 * internal streams and join back).  Results are identical to ss_render_dev on the same items.  The pointers in
 * `items` and the values behind bounds_host must stay valid and unchanged while the plan lives; the contents of the
 * x / rir / out buffers may change between runs.  Device-side `bounds` / `idx` are read at run time and must satisfy the
 * same preconditions as for ss_render_dev.  A plan may hold banked sources: every ss_bank they name must outlive the
 * plan (destroy the plan first; a bank's spectra are read at every run).  A plan binds each source's window length;
 * the start is bound too unless the source names a `win_start_dev`, whose int32 is read at every run and may change
 * between runs (written in stream order before the run).  A chunk that holds such a source runs k_blocks too: 3 kernel
 * launches per chunk, plus one each for k_rir_absmax (SS_RIR_NORMALIZE) and k_rir_direct (SS_DIRECT_TARGET with raw
 * RIRs) when present.  Not thread-safe; destroy plans before their context. */
typedef struct ss_plan ss_plan;
int ss_plan_create(ss_ctx* ctx, const ss_source* items, int n_items, ss_plan** out);
int ss_plan_run(ss_plan* plan, void* stream);
int ss_plan_is_graph(const ss_plan* plan);     /* 1 once the plan runs as an instantiated CUDA graph */
void ss_plan_destroy(ss_plan* plan);

/* ---- mixtures in plans (version 105): the training step of the separation dataloader
 * (separation/look2hear/datas/movingdatamodule.py:56-126) behind a plan's crops.  At every run, after the renders of
 * every chunk have joined, the plan assembles each mixture from its own sources' outputs with the arithmetic of
 * ss_mix_dev (compute_mch_rms_dB, SIR gains of the interferers and SNR gain of the summed noise clamped at +40 dB,
 * sums), reading the mixture's SIRs and SNR from device memory at that run.  The run stays one CUDA graph launch; a plan
 * with mixtures runs 4 more kernel launches per run, whatever the number of mixtures.
 *
 * T is a stem's output length (win_len, or N for a whole stem), E = C * T, or T with SS_MIX_MONO.
 *   - Indices name entries of the `items` passed to ss_plan_create_mix, in the caller's order.  A mixture reads the
 *     reverberant `out` of each named item (a direct-path stem is not a mixture input; ss_plan_create_target below makes
 *     it a mixture's target).  A stem
 *     may appear in several mixtures (one noise stem shared by several scenes) but only once within one mixture.
 *   - SS_MIX_MONO: every stem, speakers and noises alike, is first folded to its channel mean (the dataloader's
 *     is_mono, :62-63, :76-77): at every element t, the float32 sum of its C rows in channel order 0..C-1, every add
 *     rounded on its own, then an IEEE division by C.  The same bits on every path.  torch's CPU x.mean(dim=0) does not
 *     keep one summation order for every C and length, so against it the fold agrees to a few float32 ulps, not bit
 *     for bit.
 *   - Outputs: mix (E), speakers_out (S, E) = each speaker after its gain (speaker 0's gain is 1), rms_db (S) =
 *     compute_mch_rms_dB (:29-32) of every speaker stem before its gain, after the fold with SS_MIX_MONO, rounded to
 *     float32 (-200 for a silent stem, from the 1e-20 floor).  rms_db lets a caller apply the dataloader's silence rule
 *     (:84-101, redraw when a speaker's crop is below -40 dB) by masking or redrawing, or draw the starts on the device (ss_plan_draw below).
 *   - sirs, snr (and every win_start_dev of the plan's sources) are read on the device at every run: write them on the
 *     run's stream before the run, or in an order that is guaranteed to come before it.
 * Refused at creation, before anything is allocated and with no plan created:
 *   - S or M outside 1..8, more than 65535 mixtures: SS_ERR_UNSUPPORTED;
 *   - an index outside [0, n_items), an index repeated within one mixture (among speakers and noises), stems of one
 *     mixture that differ in C or T, a NULL snr or mix, a NULL sirs with S > 1, unknown flag bits, noise_delay < 0:
 *     SS_ERR_INVALID;
 *   - a written range (mix: E floats, speakers_out: S * E floats, rms_db: S floats) that meets another range:
 *     another written range of any mixture (its own included), any mixture's sirs (S - 1 floats) or snr (1 float), or
 *     any range an item reads or writes (x, rir, out, out_direct, bounds, idx, w, win_start_dev, whole): SS_ERR_INVALID.
 * n_mixes == 0 makes ss_plan_create_mix exactly ss_plan_create. */
#define SS_MIX_MONO 1u                /* channel mean of every stem before mixing (movingdatamodule.py:62-63, 76-77) */
typedef struct {
    int32_t speakers[8];              /* indices into `items`; speaker 0 is the reference                             */
    int32_t noises[8];
    int32_t S, M;                     /* 1..8 each                                                                    */
    const float* sirs;                /* device, S - 1 floats in dB, read at every run; NULL only when S == 1          */
    const float* snr;                 /* device, 1 float in dB, read at every run                                      */
    float* mix;                       /* device, E floats: (C, T), or (T,) with SS_MIX_MONO                            */
    float* speakers_out;              /* device, S * E floats (speakers after their gains), or NULL                    */
    float* rms_db;                    /* device, S floats, or NULL                                                     */
    uint32_t flags;                   /* SS_MIX_MONO or 0                                                             */
    int32_t noise_delay;              /* 0, or overlap_audio's shift of the summed noise in elements, as in ss_mix_item */
} ss_plan_mix;
int ss_plan_create_mix(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                       ss_plan** out);

/* ---- start draws in plans (version 107): the crop start loop of the separation dataloader
 * (separation/look2hear/datas/movingdatamodule.py:81-99), which draws up to 101 starts and rejects each one while any
 * speaker's crop is below -40 dB (compute_mch_rms_dB, :29-32), keeping the last one when every draw fails - made on the
 * device at every run, from uniform variates the caller supplies.
 *   - The readers of a draw are the plan's items whose win_start_dev is the draw's `start`; len is their win_len; M is
 *     the least over the readers of (picked candidate's N) - len + 1, the picks clamped into [0, n) as k_blocks clamps
 *     them.
 *   - Try t (0 <= t < tries) has the start s_t = min(floor(u[t] * M), M - 1) in float64 (u >= 1 gives M - 1, u < 0 or
 *     NaN gives 0); speaker k is silent at s_t when 10 log10(max(1e-20, (Q_k[s_t + len] - Q_k[s_t]) / D_k)) <
 *     threshold_db, Q_k the level table (ss_pool_levels) of speaker k's picked candidate, D_k = len for a mono table
 *     and C * len otherwise.
 *   - The draw takes the first try at which no speaker is silent, or s_{tries - 1} when there is none, and writes it to
 *     `start` (and to `used` the 1-based index of that try, or 0).
 * All draws run in one kernel launch at the head of every run (the graph's first node), before anything reads a start:
 * a run with draws launches exactly one kernel more than the same plan without them.  u and the picks are read at every
 * run: write them on the run's stream, or in an order that is guaranteed to come before it.  No error bit is added: a
 * clamped pick is reported as bit 3 by k_blocks.
 * Refused at creation, before anything is allocated:
 *   - S > 8, tries > 4096, more than 16 readers, more than 65535 draws: SS_ERR_UNSUPPORTED;
 *   - S < 1, tries < 1, a NULL start or u, a threshold that is not finite, u not 8-byte or used not 4-byte aligned, a
 *     speaker index outside [0, n_items) or repeated, a speaker that is not a pooled slot of a pool with level tables or
 *     whose win_start_dev is not `start`, a reader that is not a pooled slot, readers whose win_len differ, two draws
 *     with one `start`, and a `start` or `used` range that meets any other range the plan reads or writes (other than
 *     the readers' own reads of `start`; u counts as read): SS_ERR_INVALID. */
typedef struct {
    int32_t* start;           /* device int32 that this draw's readers read (their win_start_dev); written at every run */
    const double* u;          /* device, `tries` doubles in [0, 1), read at every run                                  */
    int32_t* used;            /* device int32 or NULL: 1-based index of the accepted try, 0 if every try was silent   */
    int32_t speakers[8];      /* indices into `items`: the crops that must not be silent                               */
    int32_t S, tries;         /* 1..8; 1..4096 (the dataloader's loop is 101)                                          */
    float threshold_db;       /* -40 in the dataloader                                                                 */
} ss_plan_draw;
/* n_draws == 0 makes it ss_plan_create_mix */
int ss_plan_create_ex(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                      const ss_plan_draw* draws, int n_draws, ss_plan** out);

/* ---- dry pools: SonicSet renders 3 utterance streams per scene, but a trajectory's RIRs do not depend on what is said
 * along it: any dry utterance rendered through a banked trajectory is physically consistent.  A dry pool is a set of n
 * dry signals that pooled slots take their dry signal from, picked on the device at every run independently of the
 * trajectory pick, so that (#dry signals x #trajectories) combinations are reachable with no host work.
 *   - ss_dry_pool_create: x[i] is a DEVICE pointer (4-byte aligned) to signal i, float32, lengths[i] samples (1 <=
 *     lengths[i] <= 2^31 - 1 - 16384, the bound of ss_source.N); 1 <= n <= 2^24.  The pool (unless SS_DRY_HOST, below)
 *     references the signals, which must outlive it; their contents may change between runs, as a candidate's x may.  flags = SS_DRY_LEVELS also builds
 *     every signal's level table: Q[0] = 0, Q[n + 1] = Q[n] + (double)(x[n] * x[n]) in float64 (lengths[i] + 1 doubles,
 *     8 bytes per sample), by the scan of ss_pool_levels over the signal as a one-channel stem (whose mono fold is the
 *     signal itself), on a stream of the library's own: the signals must be complete when the call is made (synchronise
 *     the stream that wrote them), and the tables describe them as they are then.  Returns when the pool (and its
 *     tables) is in device memory.  Refused (SS_ERR_INVALID): NULL arguments, n or a length out of range, a NULL or unaligned x[i],
 *     unknown flags.
 *   - ss_dry_pick names a pooled slot of a plan (`slot`, an index into `items`), a dry pool of the plan's context and a
 *     4-byte aligned DEVICE int32 `pick_dev`, read at every run like the slot's pick.  At every run the slot renders the
 *     candidate its own pick names - bank, bounds, N, P, K, blocking, kernel variant unchanged - with dry signal
 *     pick_dev's signal of the dry pool in place of the candidate's x.  Only samples [0, N) of it are read (the read set
 *     of a pooled slot), N the picked candidate's.  A dry pick outside [0, n) is clamped into that range and
 *     ss_device_errors reports bit 4.
 *   - Bits: a dry-picked slot's stem (and its direct stem) equals ss_render_dev of the picked candidate with x = the
 *     picked signal's first N samples, with the same fixed window, bit for bit, whenever the pooled slot has the bits of
 *     ss_render_dev at all (every candidate would choose the pool's blocking on its own, see source pools).
 *   - Start draws (ss_plan_draw): a speaker with a dry pick tests the DRY crop, not the reverberant one: silent when
 *     10 log10(max(1e-20, (Q[s + len] - Q[s]) / len)) < threshold_db, Q its dry pool's table of the picked signal.  This
 *     is the dataloader's rule applied to the dry speech: no table of the rendered stem exists for a pair drawn at run
 *     time.  The gaps create_long_audio leaves between utterances are exact zeros of the dry stream, so the rule still
 *     rejects crops that fall in a gap.  M is unchanged (the readers' picked candidates' N); speakers with and without a
 *     dry pick may share a draw.  A run with dry picks from a device dry pool launches exactly as many kernels as the
 *     same plan without them.
 *   - Mixtures take dry-picked stems like any other; a static pool (noise) takes dry picks as a moving one does.
 *   - Host dry pools: with flags | SS_DRY_HOST, x[i] may be a HOST pointer (pageable or pinned) or a device pointer.  The
 *     pool copies every signal into one pinned, mapped arena it owns (each at a 64-byte boundary, zero-padded to a whole
 *     number of float4s; 64-bit offsets), so the caller's buffers need not outlive the call.  With SS_DRY_LEVELS the
 *     tables are built as above from transient device copies of the signals, in batches of at most 256 MB (or one
 *     signal's, when larger), and kept in pinned, mapped host memory, bit for bit a device dry pool's tables; k_draw reads
 *     them over PCIe.  ss_dry_pool_bytes counts the device bytes only (the n signal pointers, and the n table pointers);
 *     ss_dry_pool_host_bytes counts the arena and the tables; ss_dry_pool_level_table returns a mapped host address.
 *     In a plan every slot with a host dry pick is staged, as a host pool's slots are: at every run k_stage reads its
 *     pick (bit 3) and its dry pick (clamped, bit 4), and copies the dry samples the picked candidate's window reads,
 *     [ws - (K + 2) * 4096, ws + win_len + 2 * 4096) clamped to [0, N), of the PICKED SIGNAL into a staging area sized
 *     once per pool and window length.  A slot of a device pool stages nothing else (its spectra stay the bank's), so a
 *     plan over device pools launches one kernel more per run than with a device dry pool; a host pool's slot stages its
 *     rows as before, so a host-pool plan launches as many kernels with host dry picks as without.  Bits, draws and
 *     errors are those of the same plan over a device dry pool of the same signals.
 * Refused by ss_plan_create_dry, before anything is allocated and with no plan created (SS_ERR_INVALID): n_picks < 0, a
 * NULL picks with n_picks > 0; a slot outside [0, n_items), or named by two dry picks; a slot that is not pooled, or
 * whose pool has loudness gains (measured with the candidates' own dry signals; ss_plan_create_pair accepts it with pair
 * gains, below), or is a host pool while the dry pool is
 * a device float32 one (k_stage copies whole float4s, which only a host or 16-bit dry pool's padded arena guarantees); a
 * NULL pool or one
 * of another context; a dry pool with a signal shorter than the slot pool's longest candidate N; a NULL or unaligned
 * pick_dev; a draw speaker with a dry pick whose dry pool has no level tables; a range a plan writes that meets a dry
 * pick or a signal of a device dry pool it uses (a host dry pool owns its arena).  A destroyed dry pool cannot be
 * detected: a dry pool must outlive every plan that uses it; ss_dry_pool_destroy waits for the device before it frees it.
 * n_picks == 0 makes ss_plan_create_dry exactly ss_plan_create_ex.  ss_version stays 108: these exports (and
 * ss_dry_pool_host_bytes for host dry pools) mark the capability. */
#define SS_DRY_LEVELS 1u
#define SS_DRY_HOST 0x100u
typedef struct {
    int32_t slot;                     /* index into `items` of a pooled slot                                           */
    const ss_dry_pool* pool;          /* the dry pool it takes its dry signal from                                     */
    const int32_t* pick_dev;          /* device int32: the signal, read at every run                                   */
} ss_dry_pick;
int ss_dry_pool_create(ss_ctx* ctx, const float* const* x, const int32_t* lengths, int n, uint32_t flags,
                       ss_dry_pool** out);
int64_t ss_dry_pool_bytes(const ss_dry_pool* pool);   /* device bytes held: n signal pointers (8 B each), and with level
                                                       * tables the tables (8 B per sample + 8, not for a host dry
                                                       * pool) and their n pointers */
int64_t ss_dry_pool_host_bytes(const ss_dry_pool* pool);   /* pinned host bytes held: the arena and the tables (0 for a
                                                            * device dry pool) */
/* Device pointer of signal i's level table (lengths[i] + 1 doubles; a mapped host address for a host dry pool), or NULL
 * without tables or with i outside [0, n). */
const double* ss_dry_pool_level_table(const ss_dry_pool* pool, int i);
void ss_dry_pool_destroy(ss_dry_pool* pool);          /* destroy dry pools after the plans that use them */
/* ---- 16-bit dry pools: a speech corpus of 16-bit PCM (LibriSpeech; SonicSet's streams place whole utterances into
 * zeros, so every sample is k / 32768 with k an int16) held as its int16 samples, about 2.125 B per sample with level
 * tables instead of 12.  A 16-bit pool behaves bit for bit as the float32 dry pool of the values k / 32768: stems,
 * direct stems, mixtures, rms_db, drawn starts, `used`, pair gains and level tables are the same, in every residency.
 *   - ss_dry_pool_create_i16: x[i] is a host or device pointer (2-byte aligned) to signal i's lengths[i] int16 samples.
 *     flags: SS_DRY_LEVELS and SS_DRY_HOST as for ss_dry_pool_create.  The pool always copies the signals into one arena
 *     it owns - device memory, or pinned, mapped host memory with SS_DRY_HOST - each at a 64-byte boundary and
 *     zero-padded to the next, so the caller's buffers may go once the call returns.
 *   - Level tables (SS_DRY_LEVELS) are kept at stride 64 (ss_dry_pool_level_stride): signal i's table holds q[j] =
 *     Q[min(64 j, lengths[i])] for j = 0..ceil(lengths[i] / 64), ceil(lengths[i] / 64) + 1 doubles, at the pool's
 *     residency; Q is the float pool's full table.  The float32 square of k / 32768 is a multiple of 2^-30 and at most
 *     1, so with lengths[i] <= 2^23 every partial sum of Q is exact in float64 in any order: Q[s] = q[s / 64] plus the
 *     float64 sum of the float32 squares of samples [64 (s / 64), s), bit for bit.  The tables are built by the scan of
 *     ss_pool_levels over transient float32 expansions of the signals, in batches of at most 256 MB of expansions.
 *   - Plans (ss_plan_create_dry / _pair): every slot with a 16-bit dry pick is staged, whatever the residency of its dry
 *     pool and its pool: at every run k_stage reads the picks (bits 3 and 4, clamped) and stores the picked signal's
 *     samples [xa & ~3, (xb + 3) & ~3) of the candidate's read set as exact float32 into the slot's staging area, sized
 *     as for a host dry pool.  A 16-bit pool serves slots of device and of host pools alike.  A draw speaker with a
 *     16-bit dry pick forms Q[s] and Q[s + len] from the sparse table and at most 63 samples each (k_draw reads them over
 *     PCIe for a host pool); speakers of float and 16-bit pools may share a draw.
 *   - Pair gains (ss_pair_gains_create) render each pair from a transient float32 expansion of the dry signal.
 *   - ss_dry_pool_bytes = 8 n (signal pointers) + the arena without SS_DRY_HOST (sum of 2 lengths[i] rounded up to 64)
 *     + with tables 8 n (table pointers) + the tables without SS_DRY_HOST (8 (ceil(lengths[i] / 64) + 1) each);
 *     ss_dry_pool_host_bytes = the arena and the tables with SS_DRY_HOST, else 0.  ss_dry_pool_level_table returns the
 *     sparse table (a mapped host address with SS_DRY_HOST).
 * Refused before anything is allocated: NULL arguments, n outside [1, 2^24], a NULL or odd x[i], unknown flags
 * (SS_ERR_INVALID); a length outside [1, 2^23] (SS_ERR_UNSUPPORTED: beyond 2^23 samples the tables' sums, and so the
 * bit contract, need not be exact).  ss_version stays 108: these exports mark the capability. */
int ss_dry_pool_create_i16(ss_ctx* ctx, const int16_t* const* x, const int32_t* lengths, int n, uint32_t flags,
                           ss_dry_pool** out);
/* Samples per level table entry of a dry pool: 1 (ss_dry_pool_create: entry s is Q[s]) or 64 (a 16-bit pool), 0 for
 * NULL. */
int ss_dry_pool_level_stride(const ss_dry_pool* pool);
/* Signal i of a 16-bit pool in its arena (a device pointer, or a host address with SS_DRY_HOST), or NULL for another
 * pool or i outside [0, n). */
const int16_t* ss_dry_pool_signal_i16(const ss_dry_pool* pool, int i);
int ss_plan_create_dry(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                       const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks, int n_picks, ss_plan** out);

/* Same, host pointers: H2D -> render -> D2H, pipelined over chunks on internal streams.  Returns
 * when every `out` is complete.  This is what the drop-in Python functions call. */
int ss_render_host(ss_ctx* ctx, const ss_source* items, int n_items);

/* Single-source conveniences with the argument order of the reference functions. */
int ss_convolve_fixed_receiver(ss_ctx* ctx, const float* source_audio, const float* rirs, float* out,
                               int32_t N, int32_t C, int32_t L);                        /* :47-61 */
int ss_convolve_moving_receiver(ss_ctx* ctx, const float* source_audio, const float* rirs,
                                const int32_t* interp_index, const float* interp_weight, float* out,
                                int32_t N, int32_t P, int32_t C, int32_t L);            /* :63-96 */

/* ---- loudness: SonicSim_audio.lufs_norm (SonicSim_audio.py:68-81) = pyloudnorm 0.1.1
 * Meter(rate, block_size).integrated_loudness + normalize.loudness.  The gating-block sample
 * bounds are computed by the caller exactly as pyloudnorm does (Python float expressions
 * truncated with int()), and passed as `brk` = the sorted distinct bounds (n_e + 1 values) plus,
 * per gating block j, the range [blk_lo[j], blk_hi[j]) of elementary intervals it covers. */
#define SS_LOUD_SCRATCH_DOUBLES 20
/* Layout: a measure-only item (out == NULL) may use any strides.  With `out`, the strides must describe a
 * dense block of N*C floats - (stride_n, stride_c) = (C, 1) for (N, C) or (1, N) for (C, N) - because
 * out[q] = gain * data[q] for q < N*C; other strides return SS_ERR_INVALID. */
typedef struct {
    const float* data;        /* element (n, c) at data[n * stride_n + c * stride_c]                   */
    float* out;               /* N*C contiguous floats = gain * data (may alias data); NULL = measure  */
    const int32_t* brk;       /* n_e + 1                                                               */
    const int32_t* blk_lo;    /* n_blocks                                                              */
    const int32_t* blk_hi;    /* n_blocks                                                              */
    double* scratch;          /* SS_LOUD_SCRATCH_DOUBLES * C * n_e doubles                             */
    double* result;           /* 2 doubles: integrated loudness (LUFS, may be -inf), linear gain       */
    int64_t stride_n, stride_c;
    int32_t N, C, n_e, n_blocks;
    double rate;              /* sample rate                                                           */
    double block_size;        /* T_g in seconds (0.4, or N / rate for short clips, SonicSim_audio.py:69) */
    double target_lufs;       /* `norm` of lufs_norm                                                   */
} ss_loud_item;

/* Device pointers, asynchronous on `stream`; all items share one sample rate; C <= 8 (channel gains
 * 1, 1, 1, 1.41, 1.41, then 1 for channels 5-7), else SS_ERR_UNSUPPORTED; at most 65535 items per call
 * (more: SS_ERR_UNSUPPORTED, before any copy or launch). */
int ss_loudness_dev(ss_ctx* ctx, const ss_loud_item* items, int n_items, void* stream);

/* One stem in host memory, N*C floats in a dense (N, C) or (C, N) layout given by the strides (other
 * strides return SS_ERR_INVALID, even when measuring only: the block is copied as it is); returns when
 * `out` (if given, same layout), the measured loudness and the linear gain are available.  A NULL brk, and
 * gating arguments that the checks of ss_post_lufs below refuse, return SS_ERR_INVALID. */
int ss_lufs_norm_host(ss_ctx* ctx, const float* data, float* out, int32_t N, int32_t C,
                      int64_t stride_n, int64_t stride_c, double rate, double block_size,
                      double target_lufs, const int32_t* brk, int32_t n_e, const int32_t* blk_lo,
                      const int32_t* blk_hi, int32_t n_blocks, double* loudness, double* gain);

/* Optional per-source post-processing of ss_render_host_ex: measure the rendered (C, N) stem and
 * normalise it to `target_lufs` on the device before it is copied out (SonicSet.py:97-101 applies
 * get_lufs_norm_audio to every stem right after rendering it).  brk == NULL skips the source.
 * An array of entries is refused (SS_ERR_INVALID, before anything is copied) unless every entry with a
 * brk has non-NULL blk_lo and blk_hi, n_e > 0, n_blocks >= 0, rate > 0 and block_size > 0 (NaN is
 * refused), and the rate of the first entry that has a brk. */
typedef struct {
    const int32_t* brk; const int32_t* blk_lo; const int32_t* blk_hi;   /* host arrays, see ss_loud_item */
    int32_t n_e, n_blocks;
    double rate, block_size, target_lufs;
    double* result;           /* host, 2 doubles: measured LUFS, linear gain (may be NULL)             */
} ss_post_lufs;

/* ss_render_host + optional loudness normalisation of each stem while it is still in HBM.  Every source
 * with a target must have C <= 8, and `post` must pass the checks of ss_post_lufs; otherwise the call
 * returns SS_ERR_INVALID before anything is copied. */
int ss_render_host_ex(ss_ctx* ctx, const ss_source* items, int n_items, const ss_post_lufs* post);

/* ---- loudness gains of a pool (version 108): SonicSet's files hold every stem loudness-normalised over the whole stem
 * (SonicSet.py:97-101, get_lufs_norm_audio: speakers to U(-19, -15) LUFS, the noise to U(-26, -22), the music to
 * U(-31, -27)), and the dataloader crops those files.  A candidate is fixed when its pool is built, so its whole-stem
 * loudness is a constant: measured here once, it makes every pooled slot that picks the candidate render the crop of the
 * normalised stem, with no loudness kernel in any plan run.
 *   - post: n entries, one per candidate, as for ss_render_host_ex (host gating plan brk / blk_lo / blk_hi, rate,
 *     block_size, target_lufs, result).  brk == NULL leaves that candidate unmeasured, with gain 1.
 *   - Every measured candidate is rendered whole, exactly as ss_pool_levels renders it (same groups, same transient
 *     buffer), and measured by the launches of ss_loudness_dev (k_kweight, k_kw_scan, k_loud_gate, -inf LUFS measured as
 *     -40): result[0..1] receives the float64 loudness and gain that ss_render_host_ex returns for the candidate rendered
 *     on its own with that target.
 *   - The pool keeps (float)gain per candidate in device memory (n floats, in ss_pool_bytes).  A pooled slot that picks
 *     candidate i stores every sample of its reverberant and of its direct stem as y * (float)gain_i, one float32
 *     multiply rounded once - the arithmetic of k_loud_scale, and the direct stem takes the reverberant stem's gain, as
 *     in ss_render_host_ex.  The gain is fused into the render kernels' stores (k_blocks reads it with the pick): a plan
 *     over pools with gains launches as many kernels per run as the same plan over the same pools without them.
 *   - ss_pool_levels afterwards builds the tables of the normalised stems (each stem scaled by (float)gain with
 *     k_loud_scale first), so that start draws test the crops the slots render.
 * Returns when the gains are in device memory.  Refused before anything is allocated, with the pool unchanged: a NULL
 * pool or post (SS_ERR_INVALID); C > 8 (SS_ERR_UNSUPPORTED, as ss_loudness_dev); entries that the checks of
 * ss_post_lufs refuse; a pool that already has gains or level tables, or that a plan has been created over
 * (SS_ERR_INVALID). */
int ss_pool_loudness(ss_pool* pool, const ss_post_lufs* post);   /* n entries, one per candidate */

/* ---- pair gains: a dry-picked slot (ss_dry_pick) renders a pair (dry signal d, candidate i) drawn at run time, whose
 * whole-stem loudness depends only on the pair.  A pair-gain table measures it once for every pair of a pool of n
 * candidates and a dry pool of n_dry signals, so that each dry-picked slot stores its crops at SonicSet's loudness
 * (get_lufs_norm_audio, as for ss_pool_loudness) with no loudness kernel and no extra launch in any plan run.
 *   - post: n entries, one per candidate of `pool`: its gating plan (brk / blk_lo / blk_hi, n_e, n_blocks), rate and
 *     block_size, as for ss_pool_loudness; target_lufs and result are ignored; brk == NULL leaves every pair of that
 *     candidate unmeasured.
 *   - targets: n_dry * n doubles, pair (d, i) at [d * n + i]; NaN leaves the pair unmeasured (gain 1).
 *   - results: NULL, or 2 * n_dry * n doubles that receive (LUFS, linear gain) of pair (d, i) at [2 * (d * n + i)], NaN
 *     for an unmeasured pair.
 *   - Each measured pair is candidate i rendered whole, with x = the first N samples of signal d (N the candidate's), as
 *     ss_pool_loudness renders a candidate (same groups of at most 256 MB of stems, candidate-major: a host pool's bank
 *     is copied to the device once per batch of its pairs; a host dry pool's signals are read from transient device
 *     copies), and measured by the same launches: results receive the float64 loudness and gain that ss_render_host_ex
 *     returns for the pair rendered on its own with that target.  Any residency of the pool and the dry pool works.
 *   - The table keeps (float)gain per pair in device memory (4 bytes per pair, ss_pair_gains_bytes).  It waits for the
 *     pool's banks and returns when the table is in device memory.
 * Refused before anything is allocated: NULL arguments (other than results), a pool or dry pool of another context, a
 * dry pool with a signal shorter than the pool's longest candidate N, entries that the checks of ss_post_lufs refuse, or
 * a target that is neither NaN nor finite (SS_ERR_INVALID); C > 8 or n_dry * n > 2^26 (SS_ERR_UNSUPPORTED).
 *
 * ss_plan_create_pair is ss_plan_create_dry with pair_gains: NULL (exactly ss_plan_create_dry), or n_picks entries, entry
 * k for picks[k], each a table or NULL (no pair gains).  A dry pick with a table stores every sample of its slot's
 * reverberant and direct stem as y * table[d * n + i], one float32 multiply rounded once, d the clamped dry pick and i
 * the clamped pick: k_blocks (or k_stage for a staged slot) reads the pair's gain with the picks, as it reads a pool's
 * gain, so a plan launches as many kernels per run with pair gains as without them.  The pair's gain replaces the
 * candidate's pool gain (ss_pool_loudness), never multiplies it, so such a dry pick is accepted on a pool with gains; a
 * dry pick without a table is still refused there.  Start draws (ss_plan_draw) are unchanged: they test a dry-picked
 * speaker's dry crop, so starts and `used` are the same with and without pair gains.  A table measured over another pool
 * than the slot's or another dry pool than the pick's is SS_ERR_INVALID.  A table must outlive every plan that uses it. */
int ss_pair_gains_create(ss_ctx* ctx, const ss_pool* pool, const ss_dry_pool* dry, const ss_post_lufs* post,
                         const double* targets, double* results, ss_pair_gains** out);
int64_t ss_pair_gains_bytes(const ss_pair_gains* g);       /* device bytes held: 4 per pair                            */
void ss_pair_gains_destroy(ss_pair_gains* g);              /* waits for the device, like ss_pool_destroy               */
int ss_plan_create_pair(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                        const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                        const ss_pair_gains* const* pair_gains /* NULL or n_picks entries, NULL = none */,
                        int n_picks, ss_plan** out);

/* ---- dereverberation targets in plans: the training target of separation + dereverberation (WHAMR!-style: the mix is
 * reverberant, the targets are the speakers' direct paths) and of the enhancement mixtures of configs[4].  A target of
 * mixture k receives, at every run, each of its speakers' direct-path stems (SS_DIRECT_TARGET, `out_direct`) with the
 * mixture's own treatment of that speaker:
 *     direct_out[s] = fold(out_direct of speaker s) * (float)g_s
 * with the fold of SS_MIX_MONO (or the stem as it is), the float32 gain g_s that scales speakers_out[s] (speaker 0: 1,
 * so its target is exactly its folded direct stem) and the same single rounded float32 multiply, in the same launch
 * that writes speakers_out (k_mix_write): a plan launches as many kernels per run with targets as without them.
 *   - The gains stay defined on the reverberant crops, as the dataloader defines them (movingdatamodule.py:105-124):
 *     mix, speakers_out, rms_db, the stems and the draws keep their bits, and the targets match the mix the model sees.
 *   - direct_out: device, S * E floats laid out like speakers_out ((S, C, T), or (S, T) with SS_MIX_MONO).  A direct
 *     set cut at the whole RIR (direct_taps >= L) makes the direct stem the reverberant stem's bits (SS_DIRECT_TARGET),
 *     and then direct_out equals speakers_out bit for bit.
 * ss_plan_create_target is ss_plan_create_pair with n_targets entries (n_targets == 0: exactly ss_plan_create_pair).
 * Refused at creation with SS_ERR_INVALID, before anything is allocated and with no plan created: a `mix` outside
 * [0, n_mixes) or named by two entries, n_targets < 0 or NULL targets with n_targets > 0, a NULL direct_out, a speaker
 * of that mixture without SS_DIRECT_TARGET, and a direct_out range that meets another range (ss_plan_mix's rule for
 * written ranges: the speakers' out_direct count as read).  ss_version stays 108: the export marks the capability. */
typedef struct {
    int32_t mix;                      /* index into `mixes`                                                           */
    float* direct_out;                /* device, S * E floats, written at every run                                   */
} ss_plan_target;
int ss_plan_create_target(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                          const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                          const ss_pair_gains* const* pair_gains /* NULL or n_picks entries, NULL = none */,
                          int n_picks, const ss_plan_target* targets, int n_targets, ss_plan** out);

/* ---- dry streams: SonicSet's speech streams laid out at every run (SonicSim_audio.py:231-277, create_long_audio),
 * from utterances held once in a 16-bit dry pool (ss_dry_pool_create_i16) instead of prebuilt 60 s streams.
 * A stream slot is a pooled slot whose dry signal is a layout of m entries over a 16-bit dry pool of n utterances: two
 * device int32 arrays ids[m] and offsets[m], 1 <= m <= 128, read at every run as picks and starts are.  At every run
 * the layout is walked in order with a running `end`, 0 at first:
 *   - ids[j] < 0: an empty entry, skipped (a fixed m holds a variable number of utterances);
 *   - ids[j] >= n, offsets[j] < 0 or offsets[j] < end: an invalid entry, skipped, and ss_device_errors reports bit 5;
 *   - otherwise the entry is kept: utterance ids[j] of len samples occupies [offsets[j], offsets[j] + len) of the
 *     stream and end becomes offsets[j] + len.  Touching placements are fine, overlapping ones are not.
 * The slot's dry signal is the stream's first N samples (N: the picked candidate's), zeros wherever no kept entry lies;
 * a kept entry that reaches past N is cut there.  A stream slot's stem, direct stem, mixture contributions, rms_db,
 * drawn start and `used` are, bit for bit, those of the same plan in which the slot takes an ss_dry_pick from a 16-bit
 * dry pool holding the stream assembled by the rule above to the slot pool's longest N.  In a draw, a stream speaker's
 * crop energy is summed per utterance from the dry pool's sparse tables: exact in float64, so the draw keeps those
 * bits.
 * A stream slot is always staged (k_stage), whatever the residency of its pool and of its dry pool; its staging area is
 * a dry-picked slot's.  The plan uploads the n utterance lengths of each dry pool its streams use once, into its
 * descriptor block.
 * ss_plan_create_stream is ss_plan_create_target with n_streams entries (n_streams == 0: exactly
 * ss_plan_create_target).  Refused at creation, before anything is allocated and with no plan created:
 *   - SS_ERR_INVALID: n_streams < 0 or NULL streams with n_streams > 0; a slot outside [0, n_items), not pooled, named
 *     by two streams or by a stream and a dry pick; a dry pool that is NULL, of another context or not 16-bit; m
 *     outside [1, 128]; a NULL or unaligned ids_dev / offsets_dev; a slot whose pool has loudness gains (a stream has
 *     no fixed (dry, trajectory) pair to measure); a draw speaker whose stream's dry pool has no level tables; a range
 *     the plan writes that meets ids_dev or offsets_dev.
 *   - SS_ERR_UNSUPPORTED: a slot pool whose longest candidate N exceeds 2^23 (beyond it the draws' sums need not be
 *     exact).
 * ss_version stays 108: the export marks the capability. */
typedef struct {
    int32_t slot;                     /* index into `items`: a pooled slot                                            */
    const ss_dry_pool* pool;          /* a 16-bit dry pool of the plan's context                                      */
    const int32_t* ids_dev;           /* device, m utterance ids (< 0: empty), read at every run                      */
    const int32_t* offsets_dev;       /* device, m stream offsets in samples, read at every run                       */
    int32_t m;                        /* 1..128                                                                       */
} ss_dry_stream;
int ss_plan_create_stream(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                          const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                          const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                          int n_targets, const ss_dry_stream* streams, int n_streams, ss_plan** out);

/* ---- background streams: SonicSet's noise and music beds laid out at every run (SonicSim_audio.py:279-340,
 * create_background_audio), from clips held once in a dry pool (float32 or 16-bit) instead of beds built once.
 * A bed slot is a pooled slot whose dry signal is a layout of m entries over a dry pool of n clips: four device int32
 * arrays ids[m], offsets[m], heads[m] and counts[m], 1 <= m <= 128, read at every run.  The layout is walked in order
 * with a running `end`, 0 at first:
 *   - ids[j] < 0: an empty entry, skipped;
 *   - ids[j] >= n, offsets[j] < 0, heads[j] < 0, counts[j] < 1, heads[j] + counts[j] beyond the clip's length or
 *     offsets[j] < end: an invalid entry, skipped, and ss_device_errors reports bit 5;
 *   - otherwise the entry is kept: clip samples [heads[j], heads[j] + counts[j]) occupy [offsets[j], offsets[j] +
 *     counts[j]) of the stream and end becomes offsets[j] + counts[j].
 * A dry stream (above) is the case heads[j] = 0, counts[j] = the utterance's length; both decide validity by one walk.
 * The slot's dry signal is the stream's first N samples (N: the picked candidate's), zeros wherever no kept entry lies.
 * A bed slot's stem, direct stem and mixture contributions are, bit for bit, those of the same plan in which the slot
 * takes an ss_dry_pick from a dry pool of the same sample format holding the bed assembled by the rule above to the
 * slot pool's longest N (of the same residency, or a float32 host pool over a host source pool, where a float32 device
 * dry pool is refused).  A bed slot is always staged (k_stage), over any dry pool and any source pool; its staging area
 * is a dry-picked slot's.  The plan uploads the n clip lengths of each dry pool its streams and beds use once, into its
 * descriptor block.  A bed slot may read a draw's start but is no draw speaker: the draws test speakers only.
 * ss_plan_create_bg is ss_plan_create_stream with n_bgs bed entries (n_bgs == 0: exactly ss_plan_create_stream).
 * Refused at creation with SS_ERR_INVALID, before anything is allocated and with *out untouched:
 *   - n_bgs < 0, or NULL bgs with n_bgs > 0;
 *   - a slot outside [0, n_items), not pooled, named by two beds, or by a bed and a dry pick or a dry stream;
 *   - a dry pool that is NULL or of another context;
 *   - m outside [1, 128];
 *   - a NULL or unaligned ids_dev / offsets_dev / heads_dev / counts_dev;
 *   - a slot whose pool has loudness gains (a bed has no fixed (dry, trajectory) pair to measure);
 *   - a slot that is a speaker of a draw;
 *   - a range the plan writes that meets any of the four arrays.
 * ss_version stays 108: the export marks the capability. */
typedef struct {
    int32_t slot;                     /* index into `items`: a pooled slot                                            */
    const ss_dry_pool* pool;          /* a dry pool of the plan's context, float32 or 16-bit                          */
    const int32_t* ids_dev;           /* device, m clip ids (< 0: empty), read at every run                           */
    const int32_t* offsets_dev;       /* device, m stream offsets in samples, read at every run                       */
    const int32_t* heads_dev;         /* device, m first clip samples placed, read at every run                       */
    const int32_t* counts_dev;        /* device, m clip samples placed, read at every run                             */
    int32_t m;                        /* 1..128                                                                       */
} ss_bg_stream;
int ss_plan_create_bg(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                      const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                      const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                      int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                      ss_plan** out);

/* ---- loudness slots: a stream or bed slot stored at SonicSet's loudness (SonicSet.py:97-101, get_lufs_norm_audio over
 * the whole 60 s stem), measured at every run.  A stream or bed has no fixed (dry signal, trajectory) pair to measure
 * once, so the plan renders the slot's whole stem at every run and measures it there.  At every run, inside the plan's
 * single graph launch, a loudness slot:
 *   1. renders its whole stem [0, N) - the picked candidate with the layout of that run - into plan-owned scratch,
 *      through the staging (k_stage) and render kernels every pooled slot uses (the slot's window is not rendered);
 *   2. measures it with the launches of ss_loudness_dev (k_kweight, k_kw_scan) over gating tables uploaded once;
 *   3. k_loud_gate<true> reads *target_dev and computes (LUFS, gain) with the float64 arithmetic of ss_render_host_ex
 *      (-inf LUFS is gained as -40) into result_dev, or plan scratch without one;
 *   4. k_loud_crop writes the slot's crop as whole[:, start : start + win_len] * (float)gain, one float32 multiply
 *      rounded once (k_loud_scale's arithmetic), and the direct-path crop of a slot with SS_DIRECT_TARGET with the same
 *      gain.  The start is the slot's (win_start, or *win_start_dev clamped into [0, N - win_len]: bit 2).
 * So the stem and direct stem of every run equal, bit for bit, the crop at that start of ss_render_host_ex of the
 * picked candidate with the stream or bed assembled by that run's layout and target_lufs = *target_dev, and result_dev
 * receives what that call's result receives.  A non-finite target stores the slot unscaled (gain 1), its result is
 * (LUFS, NaN) and ss_device_errors reports bit 6.  Draws, mixtures, rms_db and dereverberation targets read the
 * normalised crops; the draws still test a stream speaker's dry crop, so starts and `used` keep their bits.
 * Order within a run: draws, staging and renders, the six measuring launches, k_loud_crop, then the mixtures: a plan
 * with loudness slots launches 7 kernels per run more than the same plan without them, plus one launch group (k_blocks,
 * k_prepare, k_render) for every further chunk its whole stems take under the chunk budget (ss_set_chunk_bytes).  A
 * plan without loudness slots launches exactly as ss_plan_create_bg's.  Scratch, allocated at creation: per slot C * N
 * floats (twice that with SS_DIRECT_TARGET), SS_LOUD_SCRATCH_DOUBLES * C * n_e doubles and, without result_dev, two
 * doubles; and the gating tables, once per distinct plan.
 *   - gating: the slot's gating plan over N samples (brk / blk_lo / blk_hi, n_e, n_blocks, rate, block_size) as for
 *     ss_render_host_ex; target_lufs and result are ignored.  Every entry has one rate.
 *   - target_dev: device, one double, read at every run.  result_dev: NULL, or device, two doubles written at every run.
 * ss_plan_create_lufs is ss_plan_create_bg with n_lufs entries (n_lufs == 0: exactly ss_plan_create_bg).  Refused at
 * creation, before anything is allocated and with *out untouched:
 *   - SS_ERR_INVALID: n_lufs < 0 or NULL lufs with n_lufs > 0; a slot outside [0, n_items), that is not a stream or bed
 *     slot (ss_dry_stream, ss_bg_stream) or is named twice; a NULL brk, entries that the checks of ss_post_lufs refuse,
 *     a brk that is not ascending from 0 with brk[n_e] <= N, or a gating block outside [0, n_e]; a NULL or unaligned
 *     target_dev, an unaligned result_dev; a result_dev range that meets anything else the plan reads or writes;
 *   - SS_ERR_UNSUPPORTED: a slot of a host pool (SS_BANK_HOST, spectra or taps: a whole stem would stage every bank
 *     row over PCIe at every run), a slot pool whose candidates differ in N, C > 8.
 * ss_version stays 108: the export marks the capability. */
typedef struct {
    int32_t slot;                     /* index into `items`: a stream or bed slot                                     */
    ss_post_lufs gating;              /* host gating plan of the slot's N; target_lufs and result ignored             */
    const double* target_dev;         /* device, the target LUFS, read at every run                                  */
    double* result_dev;               /* device, (LUFS, gain) written at every run, or NULL                          */
} ss_stream_lufs;
int ss_plan_create_lufs(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                        const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                        const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                        int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                        const ss_stream_lufs* lufs, int n_lufs, ss_plan** out);

/* ---- layout draws: a plan draws the layouts of its stream and bed slots itself at every run, by the rules of
 * create_long_audio (SonicSim_audio.py:231-277) and create_background_audio (:279-340), instead of reading layouts
 * the caller refreshed before the run.  At the head of every run, before the start draws, one kernel launch (k_layout,
 * one warp per draw) writes each drawn slot's own layout arrays (ids_dev, offsets_dev and a bed's heads_dev, counts_dev
 * of its ss_dry_stream or ss_bg_stream); staging, draws, loudness slots and mixtures then read them as they read any
 * layout, and they hold that run's layout after it.  The layouts match the rules in distribution (the docstrings of
 * dry.long_audio_layouts and dry.background_audio_layouts), not in the reference's `random` draws.
 * Random stream (ss_phases.cuh states it once): Philox4x32-10 keyed by the 64-bit seed; block b of draw r (the entry's
 * index in `layouts`) at counter t is philox(ctr = (b, r, t_lo, t_hi), key = (seed_lo, seed_hi)), its 4 words consumed
 * in order; a uniform integer in [0, k) takes the next two words as x = w0 | w1 << 32 and is umulhi64(x, k).
 * rng_dev holds (seed, t), two int64 read at every run and never written: the same pair draws the same layouts, bit for
 * bit; a training step bumps t (rng[1] += 1) before the run.  Per row, in the order its words are drawn:
 *   - selection, a sparse Fisher-Yates order over the pool's n lengths: a stream takes utterances while the running
 *     total is below 0.9 * total and stops at the first that would overflow `total` (get_random_wav_path); a bed takes
 *     clips while the running total of select_lengths (NULL: the clip lengths) is below 0.4 * total, and the clip that
 *     reaches `total` is taken and ends it (get_random_wav_path_from_json);
 *   - placement, the selected ids in a fresh uniform order (a partial Fisher-Yates) while the cursor is below `total`:
 *     a stream draws a gap in {0, ..., 10 * sample_rate} before each utterance and places it while cursor + gap + len
 *     <= total; a bed draws a tail in {0, ..., 10 * sample_rate} after each clip, and the first clip whose length plus
 *     tail reaches the remaining samples is the end clip: slack = floor((total - cursor) * 0.1), lead and trail uniform
 *     in {0, ..., slack}, kept at cursor + lead with head lead and count min(len, total - trail - cursor) - lead when
 *     that count is above 0;
 *   - the first m entries in stream order, then -1 in every array.
 * K, the most one row can select, is worked out at creation from the pool's lengths: for a stream the largest k whose
 * k shortest utterances fit in `total` (at least 1, dry.long_audio_max_selected); for a bed the most clips whose
 * select_lengths stay below 0.4 * total, plus the one that crosses it (at most n).  A row's scratch is a hash map of
 * 2K to 4K entries and K ids in shared memory.
 * ss_plan_create_layout is ss_plan_create_lufs with n_layouts entries (n_layouts == 0: exactly ss_plan_create_lufs); a
 * plan with layout draws launches one kernel per run more.  Refused at creation, before anything is allocated and with
 * *out untouched:
 *   - SS_ERR_INVALID:
 *     - n_layouts < 0, or NULL layouts with n_layouts > 0;
 *     - a slot that is not a stream or bed slot (ss_dry_stream, ss_bg_stream), or that two entries name;
 *     - a NULL or unaligned (8 bytes) rng_dev;
 *     - total < 1, sample_rate < 1 or 10 * sample_rate above INT32_MAX;
 *     - select_lengths on a stream slot, or a negative select_lengths entry;
 *     - an rng_dev range that meets a range the plan writes;
 *     - a drawn slot's layout arrays meeting any other range the plan reads or writes, another slot's layout included.
 *   - SS_ERR_UNSUPPORTED: K above 1024.
 * ss_version stays 108: the export marks the capability. */
typedef struct {
    int32_t slot;                     /* index into `items`: a stream or bed slot                                     */
    const int64_t* rng_dev;           /* device, (seed, t), read at every run                                         */
    int32_t total;                    /* samples of the stream create_long_audio / create_background_audio would build */
    int32_t sample_rate;              /* gaps and tails are uniform in {0, ..., 10 * sample_rate}                     */
    const int32_t* select_lengths;    /* host, n entries; bed slots only; NULL = the clip lengths                     */
} ss_layout_draw;
int ss_plan_create_layout(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                          const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                          const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                          int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                          const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts, int n_layouts,
                          ss_plan** out);

/* ---- value draws: a plan writes the per-run values its slots, start draws, mixtures and loudness slots read (picks,
 * dry picks, win_start_dev, sirs, snr, a draw's u, loudness targets) itself, at the head of every run, instead of
 * reading values the caller refreshed before the run: the dataloader's random.choice of a scene, random.sample of its
 * speakers, randint crop starts, SIR ~ U(-6, 6), SNR ~ U(10, 20) and loudness targets, from one counter.  One kernel
 * launch (k_values, one warp per row) runs first in the run, before the layout draws and the start draws; everything
 * after it reads the tensors it wrote as it reads them today.  The values match the rules in distribution, not torch's
 * or `random`'s bits.
 * Random stream (ss_phases.cuh states it once), the generator and key of ss_layout_draw: element j of row b of value
 * draw r (its index in `values`) at counter t takes block philox(ctr = (b, 0x80000000 | r << 11 | j >> 1, t_lo, t_hi),
 * key = (seed_lo, seed_hi)) and its words 2 (j & 1) and 2 (j & 1) + 1 as x = w0 | w1 << 32.  Layout draws use c1 = r
 * < 2^31, so the two streams never share a block, and a plan's layout bits do not change when value draws are added.
 *   - SS_VALUE_F64: u = (x >> 11) * 2^-53; SS_VALUE_F32: u = (x >> 40) * 2^-24; v = low + (high - low) * u in double
 *     (product and sum rounded separately), rounded once to the output type; a result that is not below high becomes
 *     the largest value of the type below high;
 *   - SS_VALUE_INT: ilow + umulhi64(x, ihigh - ilow);
 *   - SS_VALUE_DISTINCT: each row an ordered sample without replacement (random.sample) from [ilow, ihigh): a partial
 *     Fisher-Yates over [0, n), n = ihigh - ilow, element j taking y = umulhi64(x_j, n - j), pos = j + y, writing
 *     ilow + a[pos] and setting a[pos] = a[j], a the identity;
 *   - base >= 0: the value is out_base[b] * stride + value, in int64 (out_base: the out of entry `base`, one int32 per
 *     row), e.g. speakers of scene-major pools: picks[b, j] = scene[b] * 3 + sample.
 * rng_dev holds (seed, t), read at every run and never written: the same pair draws the same values, bit for bit.
 * ss_plan_create_values is ss_plan_create_layout with n_values entries (n_values == 0: exactly ss_plan_create_layout);
 * a plan with value draws launches one kernel per run more.  Refused at creation, before anything is allocated and with
 * *out untouched:
 *   - SS_ERR_INVALID:
 *     - n_values < 0, or NULL values with n_values > 0; an unknown kind;
 *     - a NULL or misaligned out (4 bytes; 8 for SS_VALUE_F64) or rng_dev (8 bytes);
 *     - rows outside [1, 65535] or different from the first entry's; k outside [1, 4096];
 *     - real kinds: non-finite low or high, low >= high, a base; SS_VALUE_F32 bounds not representable in float32;
 *     - int kinds: ilow >= ihigh; SS_VALUE_DISTINCT with k > 64 or k > ihigh - ilow;
 *     - a base that is not an earlier int kind entry with k = 1; stride < 1 with a base; an int32 overflow of
 *       out_base * stride + value possible over the base entry's values;
 *     - an out that meets another entry's out, any rng_dev, or any range the plan reads or writes other than the small
 *       per-run inputs: items' pick_dev and win_start_dev (not one a start draw writes), dry picks' pick_dev, mixtures'
 *       sirs and snr, start draws' u, loudness slots' target_dev;
 *     - an rng_dev that meets a range the plan writes.
 *   - SS_ERR_UNSUPPORTED: more than 2^20 entries.
 * ss_version stays 108: the export marks the capability. */
enum { SS_VALUE_F32 = 0, SS_VALUE_F64 = 1, SS_VALUE_INT = 2, SS_VALUE_DISTINCT = 3 };
typedef struct {
    void* out;                        /* device, rows x k (row-major) float / double / int32, written at every run    */
    const int64_t* rng_dev;           /* device, (seed, t), read at every run                                         */
    int32_t kind;                     /* SS_VALUE_*                                                                   */
    int32_t rows;                     /* B, the same in every entry                                                   */
    int32_t k;                        /* elements per row                                                             */
    int32_t base;                     /* int kinds: index of an earlier int entry with k = 1, or -1                   */
    double low, high;                 /* real kinds: [low, high)                                                      */
    int32_t ilow, ihigh;              /* int kinds: [ilow, ihigh)                                                     */
    int32_t stride;                   /* with a base: >= 1                                                            */
} ss_value_draw;
int ss_plan_create_values(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                          const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                          const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                          int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                          const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts, int n_layouts,
                          const ss_value_draw* values, int n_values, ss_plan** out);

/* ---- speaker groups of layout draws: SonicSet builds every speech stream from one LibriSpeech speaker's utterances
 * (create_long_audio(audio_path, 60) over a speaker directory, SonicSim_audio.py:243; SonicSet.py:198 picks three
 * different speakers per scene).  A grouped layout draw lays its stream slot out from one contiguous group of its
 * pool's utterances, named at every run by a device int32, instead of from the whole pool.
 * Rule and random stream (ss_phases.cuh states it once): the pool's n utterances are split into G >= 1 groups by host
 * bounds 0 = bounds[0] < bounds[1] < ... < bounds[G] = n.  At every run the draw reads g from group_dev:
 *   - g outside [0, G) is clamped into range and ss_device_errors reports bit 7;
 *   - the row is exactly the ungrouped draw r (ss_layout_draw above) over a pool holding only utterances
 *     [bounds[g], bounds[g + 1]) in order: the same Philox blocks (b, r, t_lo, t_hi), the same words in the same order;
 *     every id it writes is offset by bounds[g];
 *   - reading g consumes no words.
 * So G = 1 is the ungrouped draw, and group g over the whole pool is the ungrouped draw over that group's sub-pool with
 * its ids shifted.  A value draw (SS_VALUE_DISTINCT over [0, G)) may write group_dev: the scene's S distinct speakers of
 * np.random.choice(speech_list, S, replace=False).  K (the most a row can select) is the largest K of the groups.
 * Stream slots only: SonicSet's beds draw from the split's whole clip JSON.
 * ss_plan_create_groups is ss_plan_create_values with n_grouped entries (n_grouped == 0: exactly
 * ss_plan_create_values).  A plan with grouped draws launches as many kernels per run as the same plan without groups
 * (k_layout_grouped instead of k_layout).  Refused at creation, before anything is allocated and with *out untouched:
 *   - SS_ERR_INVALID:
 *     - n_grouped < 0, or NULL groups with n_grouped > 0;
 *     - a layout index outside [0, n_layouts), or one that two entries name;
 *     - the draw of a bed slot;
 *     - n_groups < 1, NULL bounds, or bounds that do not ascend strictly from 0 to the pool's n;
 *     - a NULL or misaligned (4 bytes) group_dev;
 *     - a group_dev that meets a range the plan writes other than a value draw's out.
 *   - SS_ERR_UNSUPPORTED: K above 1024 in any group.
 * ss_version stays 108: the export marks the capability. */
typedef struct {
    int32_t layout;                   /* index into `layouts`: the draw of a stream slot                              */
    int32_t n_groups;                 /* G >= 1                                                                       */
    const int32_t* bounds;            /* host, G + 1 entries, 0 = bounds[0] < ... < bounds[G] = the pool's n          */
    const int32_t* group_dev;         /* device, one int32 read at every run                                          */
} ss_layout_group;
int ss_plan_create_groups(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                          const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                          const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                          int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                          const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts, int n_layouts,
                          const ss_value_draw* values, int n_values, const ss_layout_group* groups, int n_grouped,
                          ss_plan** out);

/* ---- trajectories of pooled slots: SonicSet times every stem's path anew (setup_dynamic_interp, SonicSim_moving.py
 * :15-45), and the same RIRs serve the path walked backwards or a contiguous stretch of it.  A trajectory entry makes a
 * pooled slot of a moving device pool render, at every run, the path its two device arrays hold over its picked
 * candidate of P positions and N samples:
 *   - path_dev: 3 int32 (a, b, dir), 0 <= a < b <= P - 1; dir 0 visits positions a, a + 1, ..., b (forward), dir 1
 *     visits b, b - 1, ..., a (reverse);
 *   - bounds_dev: p_max int32 (p_max: the pool's largest P), of which the first b - a + 1 are the visited path's
 *     cumulative segment bounds in SS_MOVING_BOUNDS form (0 first, N last, non-decreasing).
 * The slot renders visited position j with bank position a + j (forward) or b - j (reverse) and these bounds; its dry
 * signal, window, direct stem, dry pick, stream or bed stay as they are.  (0, P - 1, 0) with the candidate's own bounds
 * renders bit for bit what the slot renders without the entry, and a forward (a, b) with bounds B what the candidate
 * renders with bounds that are B over [a, b] and empty elsewhere.  An invalid path or bounds table renders the
 * candidate's own forward path and bounds, and ss_device_errors reports bit 8.  A loudness slot (ss_stream_lufs)
 * measures its whole stem with the run's trajectory.  The slot's block table, work items and dry spectra are sized for
 * any bounds table of at most P - 1 segments of any candidate (ss_phases.cuh, traj_table_cap).
 * ss_plan_create_traj is ss_plan_create_groups with n_trajs entries (n_trajs == 0: exactly ss_plan_create_groups; a
 * plan with trajectories launches as many kernels per run as without).  Refused at creation, before anything is
 * allocated and with *out untouched:
 *   - SS_ERR_INVALID:
 *     - n_trajs < 0, or NULL trajs with n_trajs > 0;
 *     - a slot outside [0, n_items), one that two entries name, or one that is not a pooled slot of a moving pool;
 *     - a pool with loudness gains (ss_pool_loudness) or a dry pick with pair gains: both were measured with the
 *       candidates' own timing;
 *     - a start draw's speaker that renders its candidate's own dry signal (its level table is that stem's);
 *     - a NULL or misaligned (4 bytes) path_dev or bounds_dev, or one that meets any other range the plan reads or
 *       writes.
 *   - SS_ERR_UNSUPPORTED: a slot of a host pool (SS_BANK_HOST), whose staging is sized from the host bounds.
 * Capability marker: the export ss_plan_create_traj.  A library that exports it takes trajectories; ss_version stays
 * 108, which callers of the earlier exports compare against, so it does not mark this capability. */
typedef struct {
    int32_t slot;                     /* index into `items`: a pooled slot of a moving device pool                   */
    const int32_t* path_dev;          /* device, (a, b, dir), read at every run                                       */
    const int32_t* bounds_dev;        /* device, p_max int32, the first b - a + 1 read at every run                   */
} ss_trajectory;
int ss_plan_create_traj(ss_ctx* ctx, const ss_source* items, int n_items, const ss_plan_mix* mixes, int n_mixes,
                        const ss_plan_draw* draws, int n_draws, const ss_dry_pick* picks,
                        const ss_pair_gains* const* pair_gains, int n_picks, const ss_plan_target* targets,
                        int n_targets, const ss_dry_stream* streams, int n_streams, const ss_bg_stream* bgs, int n_bgs,
                        const ss_stream_lufs* lufs, int n_lufs, const ss_layout_draw* layouts, int n_layouts,
                        const ss_value_draw* values, int n_values, const ss_layout_group* groups, int n_grouped,
                        const ss_trajectory* trajs, int n_trajs, ss_plan** out);

/* ---- mixture assembly of the training dataloader: separation/look2hear/datas/movingdatamodule.py
 * :29-32 (compute_mch_rms_dB) and :105-124 (SIR gains of the interferers, SNR gain of the summed noise,
 * both clamped at +40 dB, sums).  E = elements per stem (channels * samples). */
typedef struct {
    const float* speakers;    /* (S, E)  speaker_wav, speaker 0 is the reference                         */
    const float* noises;      /* (M, E)  noise_wav                                                        */
    const float* sirs;        /* (S - 1) SIR of each interferer in dB (reference: U(-6, 6))              */
    float* mix;               /* (E)     mix_wav                                                          */
    float* speakers_out;      /* (S, E)  speakers after their gains (may alias speakers; NULL = skip)    */
    double* scratch;          /* ss_mix_scratch_doubles() doubles                                        */
    int64_t E;
    int32_t S, M;
    float snr;                /* dB (reference: U(10, 20); enhancement variant U(-10, 15))               */
    int32_t noise_delay;      /* 0, or overlap_audio's shift D in elements applied to the summed noise:
                                 n[e] = (s[e-D] + s[e+D]) + s[e]  (enhancement/.../movingdatamodule.py:34-48,240) */
} ss_mix_item;

/* Limits, each checked before any copy or launch, with the outputs left untouched:
 *   - 1 <= S <= 8 and 1 <= M <= 8 (more: SS_ERR_UNSUPPORTED); sirs may be NULL only when S == 1, and
 *     E <= UINT64_MAX / 32, so that every range's byte size is representable (SS_ERR_INVALID);
 *   - ss_mix_dev takes at most 65535 items per call (more: SS_ERR_UNSUPPORTED);
 *   - within an item, every range the call writes - mix (E floats), scratch and a separate speakers_out (S * E
 *     floats) - overlaps no other range of the item (speakers, noises, sirs, mix, scratch, speakers_out); the one
 *     exception is speakers_out == speakers exactly, which scales the speakers in place (SS_ERR_INVALID);
 *   - across items (not checked): no item writes into a range another item of the same call reads or writes, and
 *     every item has its own scratch. */
int64_t ss_mix_scratch_doubles(void);
int ss_mix_dev(ss_ctx* ctx, const ss_mix_item* items, int n_items, void* stream);      /* device pointers, async */
int ss_mix_host(ss_ctx* ctx, const float* speakers, const float* noises, const float* sirs, float snr,
                float* mix, float* speakers_out, int32_t S, int32_t M, int64_t E);      /* host pointers */
int ss_mix_host_ex(ss_ctx* ctx, const float* speakers, const float* noises, const float* sirs, float snr,
                   float* mix, float* speakers_out, int32_t S, int32_t M, int64_t E, int32_t noise_delay);

/* overlap_audio (enhancement/look2hear/datas/movingdatamodule.py:34-48): y[r][n] = (x[r][n-D] + x[r][n+D]) + x[r][n],
 * zeros outside [0, T).  [x, x + rows * T) and [y, y + rows * T) must not overlap (SS_ERR_INVALID: a thread would
 * read x[n +- D] that another thread is writing); rows <= 65535 (more: SS_ERR_UNSUPPORTED). */
int ss_overlap_dev(ss_ctx* ctx, const float* x, float* y, int32_t rows, int64_t T, int64_t delay, void* stream);
int ss_overlap_host(ss_ctx* ctx, const float* x, float* y, int32_t rows, int64_t T, int64_t delay);

/* ---- dry-stream assembly: the arithmetic of SonicSim_audio.create_long_audio (SonicSim_audio.py:231-279) and
 * create_background_audio (:281-340) once the host has drawn the clips and their places (`random` stream as in the
 * reference): resampling with torchaudio.transforms.Resample's polyphase filter bank (:253-256), stereo -> mono mean
 * (:311-312) and `long_audio[:, a:b] += clip[...]` (:268, :326, :332), one kernel, the stream stays in HBM. */
typedef struct {
    const float* src;         /* (channels, src_len) device: the decoded clip at its own sample rate            */
    const float* kernel_t;    /* (taps, new_rate) device: Resample.kernel[:, 0, :] transposed; NULL = same rate  */
    int64_t dst_start;        /* first sample of the stream written                                             */
    int64_t src_start;        /* first sample of the (resampled, mono) clip used                                 */
    int64_t count;            /* samples added                                                                   */
    int32_t channels;         /* 1, or 2 (averaged after resampling)                                             */
    int32_t src_len;
    int32_t orig, new_rate;   /* sample rates divided by their gcd (Resample.orig_freq / gcd, new_freq / gcd)    */
    int32_t width, taps;      /* Resample.width; taps = 2 * width + orig                                         */
} ss_dry_clip;
/* zero-fills out[0, total) and adds every clip; device pointers, asynchronous on `stream`.  Before any copy or launch,
 * leaving `out` untouched: the destination ranges [dst_start, dst_start + count) of the clips must not overlap
 * (SS_ERR_INVALID: clips are added from different CTAs without atomics; touching ranges and count = 0 are fine), and
 * n_clips <= 65535 (more: SS_ERR_UNSUPPORTED). */
int ss_dry_assemble_dev(ss_ctx* ctx, const ss_dry_clip* clips, int n_clips, float* out, int64_t total, void* stream);

/* Counters since ss_create / ss_reset_stats: kernels launched and device time is NOT measured
 * here (bench.py uses CUDA events); this is the launch count bench.py reports as gpu_launches. */
int64_t ss_launch_count(const ss_ctx* ctx);
void ss_reset_stats(ss_ctx* ctx);

/* Per-kernel device timing with CUDA events recorded on the launching stream around k_spectra and
 * k_render (bench.py's roofline numbers).  ss_get_profile waits for the recorded launches, returns
 * the summed milliseconds of each kernel and the number of (k_spectra, k_render) launch pairs since
 * the previous call, and clears the record.  While profiling is on, chunks run one after the other on the
 * caller's stream behind a 0.3 ms idle kernel (so no interval contains a wait for the host), and the sums
 * are built from the median over calls of each launch position (repeat the same call to use this). */
int ss_set_profiling(ss_ctx* ctx, int on);
int ss_get_profile(ss_ctx* ctx, double* ms_spectra, double* ms_render, int64_t* n_pairs);

/* Test hook, pure host code (no CUDA call): the blocking plan of one source whose trajectory bounds are on the host
 * (`bounds_host`): blocks_out receives (start, len, p_lo, p_hi) per block, *aligned_out whether the blocks follow
 * the trajectory's waypoints (one transform each) or the 4096-sample grid.  Returns the number of blocks, or a
 * negative ss_status (SS_ERR_NOMEM: max_blocks too small).  A windowed item gets exactly the entries of its full
 * plan whose [start, start + len) meets the window, unchanged. */
int ss_debug_plan(const ss_source* item, int32_t* blocks_out, int32_t max_blocks, int32_t* aligned_out);

/* Test hook, pure host code: how a batch whose items need bytes[i] of scratch is cut into launch groups under `budget`
 * (ss_set_chunk_bytes): cuts_out receives the first item of every chunk followed by n.  Returns the number of values
 * written, or a negative ss_status (SS_ERR_NOMEM: max_cuts too small). */
int ss_debug_chunks(const int64_t* bytes, int32_t n, int64_t budget, int32_t* cuts_out, int32_t max_cuts);

/* pinned host memory helpers (cudaHostAlloc) for callers without torch */
int ss_host_alloc(void** ptr, int64_t bytes);
void ss_host_free(void* ptr);

#ifdef __cplusplus
}
#endif
#endif /* SONICSIM_B200_H_ */
