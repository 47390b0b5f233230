"""Direct-path targets (SS_DIRECT_TARGET): the definition in NumPy and the seeded cases the CPU and GPU tests share."""
import numpy as np

from oracle import sonicsim_oracle as so


def direct_path_rirs(rirs, taps):
    """Every row h[..., :] zeroed from cut = min(L, argmax|h| + taps) on (np.argmax: the first of equal maxima; an
    all-zero row peaks at 0).  Vectorised form of the per-row loop in test_cfg5_binaural_dual_render."""
    h = np.asarray(rirs, dtype=np.float32)
    L = h.shape[-1]
    cut = np.minimum(L, np.abs(h).argmax(axis=-1) + taps)
    return np.where(np.arange(L) < cut[..., None], h, np.float32(0)).astype(np.float32)


def normalized(h):
    """generate_rir_combination's `ir_output /= ir_output.abs().max()` in float32 (what SS_RIR_NORMALIZE computes)."""
    h = np.asarray(h, dtype=np.float32)
    return h / np.abs(h).max()


def special_rows(h, taps):
    """Rows that pin the edge cases of the definition, on the first rows of h (P, C, L): a tie +a, -a (the first
    wins), a peak within `taps` of the end (the cut clamps to L), an all-zero row."""
    rows = h.reshape(-1, h.shape[-1])
    L = rows.shape[1]
    a = np.float32(1.5) * np.abs(rows[0]).max()
    rows[0, L // 3], rows[0, L // 2] = a, -a
    if len(rows) > 1:
        rows[1, L - 3] = np.float32(1.5) * np.abs(rows[1]).max()
        assert L - 3 + taps > L
    if len(rows) > 2:
        rows[2] = 0
    return h


# name: (mode, P, C, L, N, taps); mode 0 static, 1 bounds, 2 (idx, w)
CASES = {
    "bounds": (1, 5, 2, 600, 20000, 40),
    "indexed": (2, 5, 3, 600, 12000, 40),
    "static1": (0, 1, 1, 1000, 10000, 40),
    "static2": (0, 1, 2, 1000, 10000, 40),
    "static3": (0, 1, 3, 1000, 10000, 40),
    "long": (1, 4, 2, 9000, 20000, 800),       # two RIR partitions, one peak placed in partition 1
}


def make_case(name):
    """(x, h (P, C, L), idx, w, bounds, taps) of a seeded case; idx / w / bounds describe the same trajectory
    (None for a static source)."""
    mode, P, C, L, N, taps = CASES[name]
    rng = np.random.default_rng(sum(map(ord, name)))
    x = so.synth_dry(rng, N)
    h = special_rows(so.synth_rirs(rng, P, C, L), taps)
    if name == "long":
        h[-1, -1, 5000] = np.float32(2.0)
    if mode == 0:
        return x, h, None, None, None, taps
    np.random.seed(len(name))
    idx, w = so.setup_dynamic_interp(so.synth_path(rng, P), N)
    bounds = np.concatenate([[0], np.cumsum(np.bincount(idx, minlength=P - 1))]).astype(np.int32)
    return x, h, idx.astype(np.int32), w, bounds, taps


def oracle_render(x, h, idx, w):
    """The reference's render of one source (static when idx is None)."""
    if idx is None:
        return so.convolve_fixed_receiver(x[None], h[0])
    return so.convolve_moving_receiver(x, h, idx, w)
