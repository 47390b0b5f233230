"""ctypes binding of include/sonicsim_b200.h (the C ABI) - plumbing only.

The shared library is built in-tree (sonicsim_b200/csrc/libsonicsim_b200.so) by `build()` with
nvcc for sm_90a (H100).  There is NO CPU fallback: if the library is missing or no CUDA device is
usable, every entry point raises.
"""
import ctypes
import os
import subprocess
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB_PATH = os.path.join(CSRC, "libsonicsim_b200.so")
SOURCES = ["ss_kernels.cu", "ss_loudness.cu", "ss_mix.cu", "ss_dry.cu"]
HEADERS = ["ss_core.cuh", "ss_phases.cuh", "ss_loud.cuh", "ss_internal.h", os.path.join("..", "..", "include", "sonicsim_b200.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]

SS_OK, SS_ERR_INVALID, SS_ERR_INDEX, SS_ERR_CUDA, SS_ERR_NOMEM, SS_ERR_UNSUPPORTED = 0, -1, -2, -3, -4, -5
SS_STATIC, SS_MOVING_BOUNDS, SS_MOVING_INDEXED = 0, 1, 2
SS_RIR_NORMALIZE, SS_DIRECT_TARGET = 1, 2
SS_BANK_HOST = 0x100
SS_BANK_TAPS = 0x200
SS_MIX_MONO = 1
SS_VALUE_F32, SS_VALUE_F64, SS_VALUE_INT, SS_VALUE_DISTINCT = 0, 1, 2, 3
SS_DRY_LEVELS = 1
SS_DRY_HOST = 0x100


class SsLoudItem(ctypes.Structure):
    """`ss_loud_item` of include/sonicsim_b200.h."""
    _fields_ = [("data", ctypes.c_void_p), ("out", ctypes.c_void_p), ("brk", ctypes.c_void_p),
                ("blk_lo", ctypes.c_void_p), ("blk_hi", ctypes.c_void_p), ("scratch", ctypes.c_void_p),
                ("result", ctypes.c_void_p), ("stride_n", ctypes.c_int64), ("stride_c", ctypes.c_int64),
                ("N", ctypes.c_int32), ("C", ctypes.c_int32), ("n_e", ctypes.c_int32), ("n_blocks", ctypes.c_int32),
                ("rate", ctypes.c_double), ("block_size", ctypes.c_double), ("target_lufs", ctypes.c_double)]


class SsMixItem(ctypes.Structure):
    """`ss_mix_item` of include/sonicsim_b200.h."""
    _fields_ = [("speakers", ctypes.c_void_p), ("noises", ctypes.c_void_p), ("sirs", ctypes.c_void_p),
                ("mix", ctypes.c_void_p), ("speakers_out", ctypes.c_void_p), ("scratch", ctypes.c_void_p),
                ("E", ctypes.c_int64), ("S", ctypes.c_int32), ("M", ctypes.c_int32), ("snr", ctypes.c_float),
                ("noise_delay", ctypes.c_int32)]


class SsPlanMix(ctypes.Structure):
    """`ss_plan_mix` of include/sonicsim_b200.h."""
    _fields_ = [("speakers", ctypes.c_int32 * 8), ("noises", ctypes.c_int32 * 8), ("S", ctypes.c_int32),
                ("M", ctypes.c_int32), ("sirs", ctypes.c_void_p), ("snr", ctypes.c_void_p), ("mix", ctypes.c_void_p),
                ("speakers_out", ctypes.c_void_p), ("rms_db", ctypes.c_void_p), ("flags", ctypes.c_uint32),
                ("noise_delay", ctypes.c_int32)]


class SsPlanTarget(ctypes.Structure):
    """`ss_plan_target` of include/sonicsim_b200.h."""
    _fields_ = [("mix", ctypes.c_int32), ("direct_out", ctypes.c_void_p)]


class SsPlanDraw(ctypes.Structure):
    """`ss_plan_draw` of include/sonicsim_b200.h."""
    _fields_ = [("start", ctypes.c_void_p), ("u", ctypes.c_void_p), ("used", ctypes.c_void_p),
                ("speakers", ctypes.c_int32 * 8), ("S", ctypes.c_int32), ("tries", ctypes.c_int32),
                ("threshold_db", ctypes.c_float)]


class SsDryPick(ctypes.Structure):
    """`ss_dry_pick` of include/sonicsim_b200.h."""
    _fields_ = [("slot", ctypes.c_int32), ("pool", ctypes.c_void_p), ("pick_dev", ctypes.c_void_p)]


class SsDryStream(ctypes.Structure):
    """`ss_dry_stream` of include/sonicsim_b200.h."""
    _fields_ = [("slot", ctypes.c_int32), ("pool", ctypes.c_void_p), ("ids_dev", ctypes.c_void_p),
                ("offsets_dev", ctypes.c_void_p), ("m", ctypes.c_int32)]


class SsBgStream(ctypes.Structure):
    """`ss_bg_stream` of include/sonicsim_b200.h."""
    _fields_ = [("slot", ctypes.c_int32), ("pool", ctypes.c_void_p), ("ids_dev", ctypes.c_void_p),
                ("offsets_dev", ctypes.c_void_p), ("heads_dev", ctypes.c_void_p), ("counts_dev", ctypes.c_void_p),
                ("m", ctypes.c_int32)]


class SsDryClip(ctypes.Structure):
    """`ss_dry_clip` of include/sonicsim_b200.h."""
    _fields_ = [("src", ctypes.c_void_p), ("kernel_t", ctypes.c_void_p), ("dst_start", ctypes.c_int64),
                ("src_start", ctypes.c_int64), ("count", ctypes.c_int64), ("channels", ctypes.c_int32),
                ("src_len", ctypes.c_int32), ("orig", ctypes.c_int32), ("new_rate", ctypes.c_int32),
                ("width", ctypes.c_int32), ("taps", ctypes.c_int32)]


class SsPostLufs(ctypes.Structure):
    """`ss_post_lufs` of include/sonicsim_b200.h."""
    _fields_ = [("brk", ctypes.c_void_p), ("blk_lo", ctypes.c_void_p), ("blk_hi", ctypes.c_void_p),
                ("n_e", ctypes.c_int32), ("n_blocks", ctypes.c_int32), ("rate", ctypes.c_double),
                ("block_size", ctypes.c_double), ("target_lufs", ctypes.c_double), ("result", ctypes.c_void_p)]


class SsStreamLufs(ctypes.Structure):
    """`ss_stream_lufs` of include/sonicsim_b200.h."""
    _fields_ = [("slot", ctypes.c_int32), ("gating", SsPostLufs), ("target_dev", ctypes.c_void_p),
                ("result_dev", ctypes.c_void_p)]


class SsLayoutDraw(ctypes.Structure):
    """`ss_layout_draw` of include/sonicsim_b200.h."""
    _fields_ = [("slot", ctypes.c_int32), ("rng_dev", ctypes.c_void_p), ("total", ctypes.c_int32),
                ("sample_rate", ctypes.c_int32), ("select_lengths", ctypes.c_void_p)]


class SsLayoutGroup(ctypes.Structure):
    """`ss_layout_group` of include/sonicsim_b200.h."""
    _fields_ = [("layout", ctypes.c_int32), ("n_groups", ctypes.c_int32), ("bounds", ctypes.c_void_p),
                ("group_dev", ctypes.c_void_p)]


class SsTrajectory(ctypes.Structure):
    """`ss_trajectory` of include/sonicsim_b200.h."""
    _fields_ = [("slot", ctypes.c_int32), ("path_dev", ctypes.c_void_p), ("bounds_dev", ctypes.c_void_p)]


class SsValueDraw(ctypes.Structure):
    """`ss_value_draw` of include/sonicsim_b200.h."""
    _fields_ = [("out", ctypes.c_void_p), ("rng_dev", ctypes.c_void_p), ("kind", ctypes.c_int32),
                ("rows", ctypes.c_int32), ("k", ctypes.c_int32), ("base", ctypes.c_int32), ("low", ctypes.c_double),
                ("high", ctypes.c_double), ("ilow", ctypes.c_int32), ("ihigh", ctypes.c_int32),
                ("stride", ctypes.c_int32)]


class SsSource(ctypes.Structure):
    """`ss_source` of include/sonicsim_b200.h."""
    _fields_ = [("x", ctypes.c_void_p), ("rir", ctypes.c_void_p), ("out", ctypes.c_void_p),
                ("bounds", ctypes.c_void_p), ("idx", ctypes.c_void_p), ("w", ctypes.c_void_p),
                ("N", ctypes.c_int32), ("P", ctypes.c_int32), ("C", ctypes.c_int32), ("L", ctypes.c_int32),
                ("mode", ctypes.c_int32), ("flags", ctypes.c_int32), ("bounds_host", ctypes.c_void_p),
                ("out_direct", ctypes.c_void_p), ("direct_taps", ctypes.c_int32),
                ("win_start", ctypes.c_int32), ("win_len", ctypes.c_int32), ("rir_bank", ctypes.c_void_p),
                ("win_start_dev", ctypes.c_void_p), ("pool", ctypes.c_void_p), ("pick_dev", ctypes.c_void_p)]


def _stale():
    if not os.path.isfile(LIB_PATH):
        return True
    t = os.path.getmtime(LIB_PATH)
    for f in SOURCES + HEADERS:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p) and os.path.getmtime(p) > t:
            return True
    return False


def build(force=False, verbose=False):
    """Compile the CUDA library for sm_90a with nvcc (cross-compiles without a GPU)."""
    if not force and not _stale():
        return LIB_PATH
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    extra = os.environ.get("SS_EXTRA_NVCC", "").split()          # experiment knobs, e.g. -DSS_RENDER_MINB=1
    cmd = [nvcc] + NVCC_FLAGS + extra + (["-Xptxas", "-v"] if verbose else []) + \
          ["-o", LIB_PATH] + [os.path.join(CSRC, s) for s in SOURCES]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n%s\n%s" % (" ".join(cmd), res.stderr))
    if verbose:
        print(res.stderr)
    return LIB_PATH


_lib = None
_lock = threading.Lock()


def load():
    """Load the library (no build here unless the .so is absent and nvcc exists)."""
    global _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.isfile(LIB_PATH):
            try:
                build()
            except Exception as e:  # no silent fallback: say exactly what is missing
                raise RuntimeError(
                    "sonicsim_b200: CUDA library %s is missing and could not be built (%s). "
                    "Run `python -c 'import __graft_entry__ as g; g.build()'`." % (LIB_PATH, e))
        lib = ctypes.CDLL(LIB_PATH)
        vp, i32, i64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64
        lib.ss_version.restype = ctypes.c_int
        lib.ss_strerror.restype = ctypes.c_char_p
        lib.ss_strerror.argtypes = [ctypes.c_int]
        lib.ss_last_cuda_error.restype = ctypes.c_int
        lib.ss_create.argtypes = [ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_destroy.argtypes = [vp]
        lib.ss_destroy.restype = None
        lib.ss_set_chunk_bytes.argtypes = [vp, i64]
        lib.ss_render_dev.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, vp]
        lib.ss_device_errors.argtypes = [vp, ctypes.POINTER(ctypes.c_uint32)]
        lib.ss_plan_create.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_mix.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                            ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_ex.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                          ctypes.c_int, ctypes.POINTER(SsPlanDraw), ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_dry.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                           ctypes.c_int, ctypes.POINTER(SsPlanDraw), ctypes.c_int,
                                           ctypes.POINTER(SsDryPick), ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_run.argtypes = [vp, vp]
        lib.ss_plan_is_graph.argtypes = [vp]
        lib.ss_plan_destroy.argtypes = [vp]
        lib.ss_plan_destroy.restype = None
        lib.ss_bank_create_dev.argtypes = [vp, vp, i32, i32, i32, i32, i32, vp, ctypes.POINTER(vp)]
        lib.ss_bank_create_host.argtypes = [vp, vp, i32, i32, i32, i32, i32, ctypes.POINTER(vp)]
        lib.ss_bank_bytes.argtypes = [vp]
        lib.ss_bank_bytes.restype = i64
        lib.ss_bank_host_bytes.argtypes = [vp]
        lib.ss_bank_host_bytes.restype = i64
        lib.ss_bank_flags.argtypes = [vp]
        lib.ss_bank_destroy.argtypes = [vp]
        lib.ss_bank_destroy.restype = None
        lib.ss_pool_create.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_pool_bytes.argtypes = [vp]
        lib.ss_pool_bytes.restype = i64
        lib.ss_pool_host_bytes.argtypes = [vp]
        lib.ss_pool_host_bytes.restype = i64
        lib.ss_pool_destroy.argtypes = [vp]
        lib.ss_pool_destroy.restype = None
        lib.ss_pool_levels.argtypes = [vp, ctypes.c_uint32]
        lib.ss_pool_loudness.argtypes = [vp, ctypes.POINTER(SsPostLufs)]
        lib.ss_pool_level_table.argtypes = [vp, ctypes.c_int]
        lib.ss_pool_level_table.restype = vp
        lib.ss_dry_pool_create.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_uint32, ctypes.POINTER(vp)]
        lib.ss_dry_pool_bytes.argtypes = [vp]
        lib.ss_dry_pool_bytes.restype = i64
        lib.ss_dry_pool_host_bytes.argtypes = [vp]
        lib.ss_dry_pool_host_bytes.restype = i64
        lib.ss_dry_pool_level_table.argtypes = [vp, ctypes.c_int]
        lib.ss_dry_pool_level_table.restype = vp
        lib.ss_dry_pool_destroy.argtypes = [vp]
        lib.ss_dry_pool_destroy.restype = None
        lib.ss_dry_pool_create_i16.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_uint32, ctypes.POINTER(vp)]
        lib.ss_dry_pool_level_stride.argtypes = [vp]
        lib.ss_dry_pool_signal_i16.argtypes = [vp, ctypes.c_int]
        lib.ss_dry_pool_signal_i16.restype = vp
        lib.ss_pair_gains_create.argtypes = [vp, vp, vp, ctypes.POINTER(SsPostLufs), vp, vp, ctypes.POINTER(vp)]
        lib.ss_pair_gains_bytes.argtypes = [vp]
        lib.ss_pair_gains_bytes.restype = i64
        lib.ss_pair_gains_destroy.argtypes = [vp]
        lib.ss_pair_gains_destroy.restype = None
        lib.ss_plan_create_pair.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                            ctypes.c_int, ctypes.POINTER(SsPlanDraw), ctypes.c_int,
                                            ctypes.POINTER(SsDryPick), vp, ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_target.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                              ctypes.c_int, ctypes.POINTER(SsPlanDraw), ctypes.c_int,
                                              ctypes.POINTER(SsDryPick), vp, ctypes.c_int, ctypes.POINTER(SsPlanTarget),
                                              ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_stream.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                              ctypes.c_int, ctypes.POINTER(SsPlanDraw), ctypes.c_int,
                                              ctypes.POINTER(SsDryPick), vp, ctypes.c_int, ctypes.POINTER(SsPlanTarget),
                                              ctypes.c_int, ctypes.POINTER(SsDryStream), ctypes.c_int,
                                              ctypes.POINTER(vp)]
        lib.ss_plan_create_bg.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPlanMix),
                                          ctypes.c_int, ctypes.POINTER(SsPlanDraw), ctypes.c_int,
                                          ctypes.POINTER(SsDryPick), vp, ctypes.c_int, ctypes.POINTER(SsPlanTarget),
                                          ctypes.c_int, ctypes.POINTER(SsDryStream), ctypes.c_int,
                                          ctypes.POINTER(SsBgStream), ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_lufs.argtypes = lib.ss_plan_create_bg.argtypes[:-1] + [ctypes.POINTER(SsStreamLufs),
                                                                                  ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_layout.argtypes = lib.ss_plan_create_lufs.argtypes[:-1] + [ctypes.POINTER(SsLayoutDraw),
                                                                                      ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_values.argtypes = lib.ss_plan_create_layout.argtypes[:-1] + [ctypes.POINTER(SsValueDraw),
                                                                                        ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_groups.argtypes = lib.ss_plan_create_values.argtypes[:-1] + [ctypes.POINTER(SsLayoutGroup),
                                                                                        ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_plan_create_traj.argtypes = lib.ss_plan_create_groups.argtypes[:-1] + [ctypes.POINTER(SsTrajectory),
                                                                                      ctypes.c_int, ctypes.POINTER(vp)]
        lib.ss_render_host.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int]
        lib.ss_render_host_ex.argtypes = [vp, ctypes.POINTER(SsSource), ctypes.c_int, ctypes.POINTER(SsPostLufs)]
        lib.ss_convolve_fixed_receiver.argtypes = [vp, vp, vp, vp, i32, i32, i32]
        lib.ss_convolve_moving_receiver.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32]
        dbl = ctypes.c_double
        lib.ss_loudness_dev.argtypes = [vp, ctypes.POINTER(SsLoudItem), ctypes.c_int, vp]
        lib.ss_lufs_norm_host.argtypes = [vp, vp, vp, i32, i32, i64, i64, dbl, dbl, dbl, vp, i32, vp, vp, i32,
                                          ctypes.POINTER(dbl), ctypes.POINTER(dbl)]
        lib.ss_mix_scratch_doubles.restype = i64
        lib.ss_mix_dev.argtypes = [vp, ctypes.POINTER(SsMixItem), ctypes.c_int, vp]
        lib.ss_mix_host.argtypes = [vp, vp, vp, vp, ctypes.c_float, vp, vp, i32, i32, i64]
        lib.ss_mix_host_ex.argtypes = [vp, vp, vp, vp, ctypes.c_float, vp, vp, i32, i32, i64, i32]
        lib.ss_overlap_dev.argtypes = [vp, vp, vp, i32, i64, i64, vp]
        lib.ss_overlap_host.argtypes = [vp, vp, vp, i32, i64, i64]
        lib.ss_dry_assemble_dev.argtypes = [vp, ctypes.POINTER(SsDryClip), ctypes.c_int, vp, i64, vp]
        lib.ss_debug_chunks.argtypes = [vp, i32, i64, vp, i32]
        lib.ss_debug_plan.argtypes = [ctypes.POINTER(SsSource), vp, i32, ctypes.POINTER(i32)]
        lib.ss_launch_count.argtypes = [vp]
        lib.ss_launch_count.restype = i64
        lib.ss_reset_stats.argtypes = [vp]
        lib.ss_reset_stats.restype = None
        lib.ss_set_profiling.argtypes = [vp, ctypes.c_int]
        lib.ss_get_profile.argtypes = [vp, ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_double),
                                       ctypes.POINTER(i64)]
        lib.ss_host_alloc.argtypes = [ctypes.POINTER(vp), i64]
        lib.ss_host_free.argtypes = [vp]
        lib.ss_host_free.restype = None
        _lib = lib
        return lib


EXPORTS = ["ss_version", "ss_strerror", "ss_last_cuda_error", "ss_create", "ss_destroy",
           "ss_set_chunk_bytes", "ss_render_dev", "ss_device_errors", "ss_plan_create", "ss_plan_create_mix", "ss_plan_create_ex", "ss_plan_run", "ss_plan_is_graph", "ss_plan_destroy", "ss_bank_create_dev", "ss_bank_create_host", "ss_bank_bytes", "ss_bank_host_bytes", "ss_bank_flags", "ss_bank_destroy", "ss_pool_create", "ss_pool_bytes", "ss_pool_host_bytes", "ss_pool_destroy", "ss_pool_levels", "ss_pool_level_table", "ss_pool_loudness", "ss_dry_pool_create", "ss_dry_pool_bytes", "ss_dry_pool_host_bytes", "ss_dry_pool_level_table", "ss_dry_pool_destroy", "ss_dry_pool_create_i16", "ss_dry_pool_level_stride", "ss_dry_pool_signal_i16", "ss_plan_create_dry", "ss_pair_gains_create", "ss_pair_gains_bytes", "ss_pair_gains_destroy", "ss_plan_create_pair", "ss_plan_create_target", "ss_plan_create_stream", "ss_plan_create_bg", "ss_plan_create_lufs", "ss_plan_create_layout", "ss_plan_create_values", "ss_plan_create_groups", "ss_plan_create_traj", "ss_render_host", "ss_render_host_ex", "ss_convolve_fixed_receiver",
           "ss_convolve_moving_receiver", "ss_loudness_dev", "ss_lufs_norm_host", "ss_mix_scratch_doubles", "ss_mix_dev", "ss_mix_host",
           "ss_mix_host_ex", "ss_overlap_dev", "ss_overlap_host", "ss_dry_assemble_dev", "ss_debug_plan", "ss_debug_chunks", "ss_launch_count", "ss_reset_stats", "ss_set_profiling", "ss_get_profile", "ss_host_alloc",
           "ss_host_free"]


def check(status):
    """Map ss_status to the exception types the reference raises (SURVEY 8b)."""
    if status == SS_OK:
        return
    lib = load()
    msg = lib.ss_strerror(status).decode()
    if status == SS_ERR_INDEX:
        raise IndexError(msg)
    if status in (SS_ERR_INVALID, SS_ERR_UNSUPPORTED):
        raise ValueError(msg)
    if status == SS_ERR_NOMEM:
        raise MemoryError(msg)
    raise RuntimeError("%s (cudaError %d)" % (msg, lib.ss_last_cuda_error()))


_ctx = {}


def default_device() -> int:
    """CUDA ordinal the process renders on when none is given: SONICSIM_B200_DEVICE, else LOCAL_RANK, else 0."""
    return int(os.environ.get("SONICSIM_B200_DEVICE", os.environ.get("LOCAL_RANK", "0")))


def context(device=None):
    """One ss_ctx per (process, device).  Raises if no CUDA device is usable."""
    lib = load()
    if device is None:
        device = default_device()
    with _lock:
        if device in _ctx:
            return _ctx[device]
        h = ctypes.c_void_p()
        st = lib.ss_create(int(device), ctypes.byref(h))
        if st != SS_OK:
            raise RuntimeError("sonicsim_b200: ss_create(device=%d) failed: %s (cudaError %d) - an H100 "
                               "(sm_90) CUDA device is required, there is no CPU fallback"
                               % (device, lib.ss_strerror(st).decode(), lib.ss_last_cuda_error()))
        _ctx[device] = h
        return h
