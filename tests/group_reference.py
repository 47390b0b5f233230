"""Grouped layout draws (ss_layout_group; render.LayoutDraw(groups=, group=)) for the tests: the bindings of the CPU
emulation tests/emu/ss_emu_layout_group.cu (k_layout_grouped's own code), the ungrouped rows of a sub-pool from
tests/emu/ss_emu_layout.cu, and corpora cut into speaker groups.  Test infrastructure."""
import ctypes

import numpy as np

from emu import build_emu
from layout_reference import load_emu as load_layout_emu
from sonicsim_b200 import dry


def load_emu():
    """lib ss_emu_layout_group, built if stale, with its entry point bound."""
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    lib = build_emu.load("ss_emu_layout_group")
    fn = lib.emu_layout_group_rows
    fn.argtypes, fn.restype = [vp, i32, i32, vp] + [i32] * 5 + [vp, i32, vp, vp, vp], ctypes.c_int
    return lib


def grouped_rows(rng_pairs, r, lengths, total, m, gap_max, bounds=None, group=None, K=None):
    """Rows of stream draw r as k_layout_grouped draws them, row q at rng_pairs[q] over group group[q] of `bounds`
    (None: ungrouped rows).  K defaults to the plan's (the largest of the groups').  Returns (ids, offsets, err): two
    (rows, m) int32 arrays and the error bits of every row."""
    L = np.ascontiguousarray(lengths, dtype=np.int32)
    rng = np.ascontiguousarray(np.asarray(rng_pairs, dtype=np.int64).reshape(-1, 2))
    rows = rng.shape[0]
    if K is None:
        K = dry.long_audio_max_selected(L, total, bounds)
    b = None if bounds is None else np.ascontiguousarray(bounds, dtype=np.int32)
    g = None if group is None else np.ascontiguousarray(np.broadcast_to(np.asarray(group, np.int32), (rows,)))
    ids, offs = np.zeros((rows, m), np.int32), np.zeros((rows, m), np.int32)
    err = load_emu().emu_layout_group_rows(rng.ctypes.data, rows, r, L.ctypes.data, L.size, m, total, gap_max, K,
                                           None if b is None else b.ctypes.data, 0 if b is None else b.size - 1,
                                           None if g is None else g.ctypes.data, ids.ctypes.data, offs.ctypes.data)
    return ids, offs, err


def plain_rows(rng_pairs, r, lengths, total, m, gap_max):
    """Ungrouped stream rows of draw r over `lengths` (tests/emu/ss_emu_layout.cu, k_layout's code), with the K of
    those lengths: (ids, offsets), (rows, m) each."""
    L = np.ascontiguousarray(lengths, dtype=np.int32)
    rng = np.ascontiguousarray(np.asarray(rng_pairs, dtype=np.int64).reshape(-1, 2))
    rows = rng.shape[0]
    ids, offs = np.zeros((rows, m), np.int32), np.zeros((rows, m), np.int32)
    load_layout_emu().emu_layout_rows(rng.ctypes.data, rows, r, L.ctypes.data, None, L.size, m, total, gap_max,
                                      dry.long_audio_max_selected(L, total), ids.ctypes.data, offs.ctypes.data, None,
                                      None)
    return ids, offs


def shifted(ids, lo):
    """ids of a sub-pool row numbered in the whole pool: every id but -1 plus lo."""
    return np.where(ids >= 0, ids + lo, ids).astype(np.int32)


def corpus(seed, sizes, lo, hi):
    """Utterance lengths of speakers with `sizes` utterances each, uniform in [lo, hi]: (lengths, bounds)."""
    rng = np.random.default_rng(seed)
    bounds = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    return rng.integers(lo, hi + 1, int(bounds[-1])).astype(np.int32), bounds
