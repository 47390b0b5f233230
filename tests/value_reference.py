"""Value draws (ss_value_draw; render.ValueDraw) restated in NumPy, for the tests: the Philox4x32-10 addressing of
include/sonicsim_b200.h, the real, integer and distinct rules, and base chains, written out independently of
ss_phases.cuh (a dense dict where the kernel keeps a hashed map), plus the binding of the emulation
(tests/emu/ss_emu_values.cu) that runs k_values' own row code.  Test infrastructure."""
import ctypes

import numpy as np

from emu import build_emu
from layout_reference import M32, M64, philox
from sonicsim_b200 import _lib

KINDS = {np.float32: _lib.SS_VALUE_F32, np.float64: _lib.SS_VALUE_F64, np.int32: _lib.SS_VALUE_INT}


def load_emu():
    """lib ss_emu_values (tests/emu/ss_emu_values.cu), built if stale, with its entry points bound."""
    vp, i32, u64, f64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint64, ctypes.c_double
    lib = build_emu.load("ss_emu_values")
    for name, argtypes, restype in (("emu_value_rows", [ctypes.POINTER(_lib.SsValueDraw), i32, i32], None),
                                    ("emu_value_word", [ctypes.c_int64, ctypes.c_int64, i32, i32, i32], u64),
                                    ("emu_value_f64", [f64, f64, u64], f64),
                                    ("emu_value_f32", [f64, f64, u64], ctypes.c_float),
                                    ("emu_value_below", [u64, u64], u64)):
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = argtypes, restype
    return lib


class Spec:
    """One value draw of a test: dtype, k, [low, high), distinct, base (index of an earlier draw), stride."""

    def __init__(self, dtype, k=1, low=0.0, high=1.0, distinct=False, base=None, stride=0):
        self.dtype, self.k, self.low, self.high = np.dtype(dtype).type, k, low, high
        self.distinct, self.base, self.stride = distinct, base, stride


def emu_rows(lib, specs, rows, seed, t, lanes=32):
    """Every draw's (rows, k) array as the emulated k_values writes it at (seed, t)."""
    rng = np.array([seed, t], dtype=np.int64)
    outs = [np.zeros((rows, s.k), s.dtype) for s in specs]
    arr = (_lib.SsValueDraw * len(specs))()
    for r, s in enumerate(specs):
        kind = KINDS[s.dtype]
        e = _lib.SsValueDraw(out=outs[r].ctypes.data, rng_dev=rng.ctypes.data, kind=kind, rows=rows, k=s.k,
                             base=-1 if s.base is None else s.base, stride=s.stride)
        if kind == _lib.SS_VALUE_INT:
            e.ilow, e.ihigh = int(s.low), int(s.high)
            if s.distinct:
                e.kind = _lib.SS_VALUE_DISTINCT
        else:
            e.low, e.high = float(s.low), float(s.high)
        arr[r] = e
    lib.emu_value_rows(arr, len(specs), lanes)
    return outs


def word(seed, t, r, b, j):
    """x of element j of row b of value draw r at (seed, t): block (b, 2^31 | r << 11 | j >> 1, t_lo, t_hi) under the
    key (seed_lo, seed_hi), words 2 (j & 1) and 2 (j & 1) + 1."""
    s, u = seed & M64, t & M64
    w = philox((b, 0x80000000 | r << 11 | j >> 1, u & M32, u >> 32), (s & M32, s >> 32))
    h = 2 * (j & 1)
    return w[h] | w[h + 1] << 32


def real64(x, low, high):
    v = low + (high - low) * ((x >> 11) * 2.0 ** -53)          # Python floats: float64, no contraction
    return v if v < high else float(np.nextafter(high, -np.inf))


def real32(x, low, high):
    v = np.float32(low + (high - low) * ((x >> 40) * 2.0 ** -24))
    return v if v < np.float32(high) else np.nextafter(np.float32(high), np.float32(-np.inf))


def below(x, n):
    return (x * n) >> 64


def rows(specs, nrows, seed, t):
    """The restatement of emu_rows."""
    outs = [np.zeros((nrows, s.k), s.dtype) for s in specs]
    for b in range(nrows):
        for r, s in enumerate(specs):
            xs = [word(seed, t, r, b, j) for j in range(s.k)]
            if s.dtype is np.float64:
                outs[r][b] = [real64(x, s.low, s.high) for x in xs]
                continue
            if s.dtype is np.float32:
                outs[r][b] = [real32(x, s.low, s.high) for x in xs]
                continue
            low, n = int(s.low), int(s.high) - int(s.low)
            add = low + (int(outs[s.base][b, 0]) * s.stride if s.base is not None else 0)
            if not s.distinct:
                outs[r][b] = [add + below(x, n) for x in xs]
                continue
            a = {}
            for j, x in enumerate(xs):                         # partial Fisher-Yates over [0, n)
                pos = j + below(x, n - j)
                outs[r][b, j] = add + a.get(pos, pos)
                a[pos] = a.get(j, j)
    return outs
