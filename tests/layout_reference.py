"""Layout draws (ss_layout_draw; render.LayoutDraw) restated in Python, for the tests: the Philox4x32-10 word stream of
include/sonicsim_b200.h and the per-row rules of k_layout (create_long_audio's and create_background_audio's), written
out independently of ss_phases.cuh (a dense Fisher-Yates array where the kernel keeps a sparse map), and the host
reference loops the layouts are compared against in distribution.  Test infrastructure."""
import ctypes
import random

from emu import build_emu
from sonicsim_b200 import dry

M32, M64 = 0xFFFFFFFF, (1 << 64) - 1


def load_emu():
    """lib ss_emu_layout (tests/emu/ss_emu_layout.cu), built if stale, with its entry points bound."""
    vp, i32 = ctypes.c_void_p, ctypes.c_int
    lib = build_emu.load("ss_emu_layout")
    for name, argtypes, restype in (("emu_philox", [vp, vp, vp], None),
                                    ("emu_rng_below", [vp, i32, vp, i32, vp], None),
                                    ("emu_layout_rows", [vp, i32, i32, vp, vp] + [i32] * 5 + [vp] * 4, None),
                                    ("emu_layout_walk", [vp] * 4 + [i32, vp, i32, vp], ctypes.c_int)):
        fn = getattr(lib, name)
        fn.argtypes, fn.restype = argtypes, restype
    return lib


def philox(ctr, key):
    """Philox4x32-10 (Salmon et al., SC'11) of a 4-word counter under a 2-word key."""
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for i in range(10):
        if i:
            k0, k1 = (k0 + 0x9E3779B9) & M32, (k1 + 0xBB67AE85) & M32
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M32, (p0 >> 32) ^ c3 ^ k1, p0 & M32
    return [c0, c1, c2, c3]


class Words:
    """The word stream of layout draw r at (seed, t): block b is philox((b, r, t_lo, t_hi), (seed_lo, seed_hi))."""

    def __init__(self, seed, t, r):
        s, u = seed & M64, t & M64
        self.key, self.ctr, self.b, self.buf = (s & M32, s >> 32), (r, u & M32, u >> 32), 0, []

    def word(self):
        if not self.buf:
            self.buf = philox((self.b,) + self.ctr, self.key)
            self.b += 1
        return self.buf.pop(0)

    def below(self, k):
        """A uniform integer in [0, k): umulhi64(w0 | w1 << 32, k)."""
        lo = self.word()
        return ((lo | self.word() << 32) * k) >> 64


def layout_row(seed, t, r, lengths, total, m, sample_rate, bed, select=None):
    """Row of layout draw r at (seed, t): (ids, offsets, heads, counts) lists of m entries (heads and counts all -1 for
    a stream), and a note of what happened: "dropped" when a bed's end clip had a count <= 0."""
    g = Words(seed, t, r)
    n, sl = len(lengths), lengths if select is None else select
    order = list(range(n))
    thr = (0.4 if bed else 0.9) * total
    acc, s = 0, 0
    while s < n and acc < thr:                                  # selection: a Fisher-Yates order, with its stop rule
        p = s + g.below(n - s)
        x = order[p]
        if not bed and acc + sl[x] > total:
            break
        order[p], order[s] = order[s], x
        s += 1
        if bed and not acc + sl[x] < total:
            break
        acc += sl[x]
    sel = order[:s]
    rows, cur, note = [], 0, None
    for j in range(s):                                          # placement: a fresh order over the selected ids
        if cur >= total or len(rows) == m:
            break
        v = j + g.below(s - j)
        sel[j], sel[v] = sel[v], sel[j]
        i, ln = sel[j], lengths[sel[j]]
        gap = g.below(10 * sample_rate + 1)
        if not bed:
            if cur + gap + ln > total:
                break
            rows.append((i, cur + gap, -1, -1))
            cur += gap + ln
        elif ln + gap >= total - cur:
            slack = int((total - cur) * 0.1)
            lead, trail = g.below(slack + 1), g.below(slack + 1)
            c = min(ln, total - trail - cur) - lead
            if c > 0:
                rows.append((i, cur + lead, lead, c))
            else:
                note = "dropped"
            break
        else:
            rows.append((i, cur, 0, ln))
            cur += ln + gap
    rows += [(-1, -1, -1, -1)] * (m - len(rows))
    return [list(v) for v in zip(*rows)], note


def walk_rule(ids, offsets, heads, counts, lengths):
    """The stream / bed walk of include/sonicsim_b200.h (heads None: a stream): (kept entries, any invalid one)."""
    kept, bad, end = 0, False, 0
    for j, (i, o) in enumerate(zip(ids, offsets)):
        if i < 0:
            continue
        h, c = (0, lengths[i]) if heads is None or i >= len(lengths) else (heads[j], counts[j])
        if i >= len(lengths) or o < 0 or o < end or h < 0 or c < 1 or h + c > lengths[i]:
            bad = True
            continue
        kept += 1
        end = o + c
    return kept, bad


def host_stream(lengths, total, sample_rate):
    """get_random_wav_path's selection on lengths, then _place_long_audio: ((id, offset), ...) in stream order."""
    cands, chosen, acc = list(range(len(lengths))), [], 0
    while cands and acc < total * 0.9:
        pick = random.choice(cands)
        if acc + lengths[pick] > total:
            break
        chosen.append(pick)
        acc += lengths[pick]
        cands.remove(pick)
    places = dry._place_long_audio([lengths[c] for c in chosen], total, sample_rate)[0]
    return tuple((chosen[k], dst) for k, dst, _, _ in places)


def host_bed(lengths, json_path, total, sample_rate):
    """get_random_wav_path_from_json (threshold 0.4, the JSON keys are clip ids) then _place_background_audio:
    ((id, offset, head, count), ...) in stream order."""
    chosen = dry.get_random_wav_path_from_json(json_path, total, threshold=0.4)
    places = dry._place_background_audio([lengths[int(p)] for p in chosen], total, total / sample_rate,
                                         sample_rate)[0]
    return tuple((int(chosen[k]), dst, src, cnt) for k, dst, src, cnt in places)
