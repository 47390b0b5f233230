"""Build the CPU emulations of the kernels with g++: tests/emu/<name>.cu into tests/emu/lib<name>.so, and load them with
the argtypes of their entry points.  Test infrastructure."""
import ctypes
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "sonicsim_b200", "csrc")

vp, i32, f32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_float
i32p = ctypes.POINTER(ctypes.c_int32)

# entry point: argtypes.  The sources include each other, so one entry point may be exported by several libraries.
ARGTYPES = {
    "emu_bank_create": [vp] + [i32] * 5 + [vp, vp],
    "emu_clamp_pick": [i32, i32, i32p],
    "emu_clamp_win_start": [i32, i32, i32, i32p],
    "emu_draw": [vp, vp, i32, vp, i32, i32, vp, i32, f32, i32p],
    "emu_draw_i16": [vp, vp, vp, vp, i32, i32, i32, vp, i32, f32, i32p],
    "emu_draw_mixed": [vp] * 9 + [i32, vp, vp, i32, i32, vp, i32, f32, i32p],
    "emu_draw_start": [ctypes.c_double, i32],
    "emu_dry_stage_slot": [vp] * 4 + [i32] * 10 + [vp] + [i32] * 4 + [vp] * 5,
    "emu_pair_heads": [vp, vp, i32, i32, i32, vp, i32, i32, i32, vp],
    "emu_pick_candidate": [i32] * 5 + [vp],
    "emu_pick_parts": [i32, i32, vp, vp, vp] + [i32] * 5 + [vp],
    "emu_pick_pooled": [vp, vp, vp, i32, vp, i32] + [i32] * 7 + [vp],
    "emu_pick_slot": [i32, i32, vp, vp, ctypes.POINTER(f32)],
    "emu_pool_table_cap": [vp, vp, vp, vp] + [i32] * 4,
    "emu_pool_table_cap_parts": [vp] * 5 + [i32] * 3,
    "emu_render_slot": [vp] * 4 + [i32] * 8,
    "emu_render_window": [vp] * 6 + [i32] * 8 + [vp] + [i32] * 3 + [vp],
    "emu_set_gain": [f32],
    "emu_sparse_levels": [vp, vp, vp, i32, vp],
    "emu_speaker_i16": [vp, vp, i32, i32, vp],
    "emu_stage_area": [i32] * 4 + [vp],
    "emu_stage_cap": [vp] * 5 + [i32] * 3 + [vp],
    "emu_stage_i16": [vp] + [i32] * 6 + [vp, vp] + [i32] * 3 + [vp, vp, vp],
    "emu_stage_set": [i32] * 4 + [vp] + [i32] * 2 + [vp],
    "emu_stage_slot": [vp] * 4 + [i32] * 10 + [vp] * 5,
    "emu_tap_bank": [vp] + [i32] * 5 + [vp, vp],
    "emu_tap_block": [ctypes.c_int64, i32, i32, vp, vp],
    "emu_tap_transform": [vp, vp] + [i32] * 7 + [vp, vp],
    "emu_window_table_cap": [vp] + [i32] * 6,
    "emu_window_tables": [vp] + [i32] * 5 + [vp],
}
VOID = {"emu_set_gain"}

_loaded = {}


def build(name="ss_emu", force=False):
    """tests/emu/lib<name>.so, rebuilt when it is older than any emulation source or library header."""
    src = os.path.join(HERE, name + ".cu")
    out = os.path.join(HERE, "lib%s.so" % name)
    deps = glob.glob(os.path.join(HERE, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh"))
    if not force and os.path.isfile(out) and all(os.path.getmtime(out) >= os.path.getmtime(d) for d in deps):
        return out
    cuda_inc = os.environ.get("CUDA_INC", "/usr/local/cuda/include")
    tmp = "%s.%d.tmp" % (out, os.getpid())
    cmd = ["g++", "-O2", "-shared", "-fPIC", "-x", "c++", "-I" + cuda_inc, "-o", tmp, src]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("g++ failed: %s\n%s" % (" ".join(cmd), res.stderr))
    os.replace(tmp, out)            # a library another process has loaded is never rewritten in place
    return out


def load(name):
    """ctypes handle of lib<name>.so, built if stale, with the argtypes of every entry point it exports."""
    if name not in _loaded:
        lib = ctypes.CDLL(build(name))
        for fn, argtypes in ARGTYPES.items():
            if hasattr(lib, fn):
                getattr(lib, fn).argtypes = argtypes
                if fn in VOID:
                    getattr(lib, fn).restype = None
        _loaded[name] = lib
    return _loaded[name]


if __name__ == "__main__":
    print(build(force=True))
