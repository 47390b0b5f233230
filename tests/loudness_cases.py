"""Loudness cases the CPU and GPU loudness tests share: signals, rates, partitions and the float64 BS.1770 reference
with its gate margins.  Test infrastructure."""
import numpy as np
import torch

from oracle import sonicsim_oracle as so

NAN = float("nan")


def stems(seed, N, C, sr=16000):
    rng = np.random.default_rng(seed)
    t = np.arange(N) / sr
    env = 0.5 + 0.5 * np.sin(2 * np.pi * 0.7 * t + rng.random() * 6)          # loud / quiet passages exercise the gates
    x = rng.standard_normal((N, C)) * env[:, None] * 0.05
    x[: N // 7] *= 1e-4                                                        # a near-silent lead-in (absolute gate)
    x += 0.02 * np.sin(2 * np.pi * 30 * t)[:, None]                            # sub-38 Hz content (high-pass matters)
    return x.astype(np.float32)


def subsonic(seed, N, C, sr=16000):
    """Noise over a strong 20 Hz tone: the 38 Hz high-pass carries a large state from one interval into the next."""
    rng = np.random.default_rng(seed)
    t = np.arange(N) / sr
    return (0.6 * np.sin(2 * np.pi * 20 * t)[:, None] + 0.05 * rng.standard_normal((N, C))).astype(np.float32)

RATES = [8000, 16000, 22050, 44100, 48000]

EXACT_DB = 1e-6           # kernels vs the float64 restatement: they differ only by float64 rounding of the filter state


def block_size_of(N, sr):
    return 0.4 if N / sr >= 0.4 else N / sr                                   # SonicSim_audio.py:69


def assert_clear_of_gates(x, sr, block, margin=1e-3):
    """No gating block of `x` is within `margin` dB of the absolute (-70) or the relative gate, so rounding cannot
    move a block across a gate and the comparison with the reference cannot turn on a near-tie."""
    l, gamma_r = so.bs1770_block_loudness(x, sr, block, up_to_8_channels=True)
    fin = l[np.isfinite(l)]
    assert np.all(np.abs(fin + 70.0) > margin), np.min(np.abs(fin + 70.0))
    if np.isfinite(gamma_r):
        assert np.all(np.abs(fin - gamma_r) > margin), np.min(np.abs(fin - gamma_r))
    return l, gamma_r


def n_samples_for(n_e, sr):
    """A clip length whose gating plan has exactly `n_e` elementary intervals (shortest such N from 0.05 s on)."""
    from sonicsim_b200.SonicSim_audio import gating_plan
    N = int(0.05 * sr)
    while True:
        brk = gating_plan(N, float(sr), float(block_size_of(N, sr)), 1)[0]
        if len(brk) - 1 == n_e:
            return N
        assert len(brk) - 1 < n_e, "no clip length at %g Hz has %d intervals" % (sr, n_e)
        N += max(1, int(0.01 * sr)) if len(brk) - 1 < n_e - 1 else 1

PARTITION_CASES = [(16000, 100001, 2, stems), (48000, int(1.06 * 48000), 7, stems), (22050, 5000, 1, stems),
                   (8000, int(0.41 * 8000), 2, subsonic), (48000, int(1.3 * 48000), 3, subsonic)]

REFINES = (1, 2, 5, 32)


def _reference(x, sr):
    return so.bs1770_integrated_loudness(x, sr, block_size_of(x.shape[0], sr), up_to_8_channels=True)


class Stem:
    """One ss_loud_item on the device.  `x` (N, C) float32; layout "nc" (interleaved) or "cn" (channel-major); `out`
    "none" (measure only), "alias" (normalised in place) or "sep" (a separate NaN-filled buffer); `off` floats in
    front of the data in its buffer (1 = not 16-byte aligned: k_loud_scale's scalar path); `refine` as gating_plan's."""

    def __init__(self, x, sr, target, layout="cn", out="sep", off=0, pad=3, refine=1):
        from sonicsim_b200.SonicSim_audio import gating_plan
        self.x, self.sr, self.target, self.layout, self.mode, self.off = x, sr, target, layout, out, off
        N, C = x.shape
        self.N, self.C, self.n = N, C, N * C
        self.block = block_size_of(N, sr)
        brk, lo, hi = gating_plan(N, float(sr), float(self.block), refine)
        dense = x.T.reshape(-1) if layout == "cn" else x.reshape(-1)
        self.buf = torch.full((off + self.n + pad,), NAN, device="cuda")
        self.buf[off:off + self.n] = torch.from_numpy(np.ascontiguousarray(dense)).cuda()
        self.obuf = torch.full_like(self.buf, NAN) if out == "sep" else None
        self.tabs = [torch.from_numpy(a.astype(np.int32)).cuda() for a in (brk, lo, hi)]
        self.scratch = torch.empty(20 * C * (len(brk) - 1), dtype=torch.float64, device="cuda")
        self.res = torch.full((2,), NAN, dtype=torch.float64, device="cuda")
        sn, sc = (1, N) if layout == "cn" else (C, 1)
        data = self.buf.data_ptr() + 4 * off
        outp = {"none": None, "alias": data, "sep": None if self.obuf is None else self.obuf.data_ptr() + 4 * off}[out]
        from sonicsim_b200 import _lib
        self.item = _lib.SsLoudItem(data=data, out=outp, brk=self.tabs[0].data_ptr(), blk_lo=self.tabs[1].data_ptr(),
                                    blk_hi=self.tabs[2].data_ptr(), scratch=self.scratch.data_ptr(),
                                    result=self.res.data_ptr(), stride_n=sn, stride_c=sc, N=N, C=C, n_e=len(brk) - 1,
                                    n_blocks=len(lo), rate=float(sr), block_size=float(self.block),
                                    target_lufs=float(target))

    def lufs_gain(self):
        r = self.res.cpu().numpy()
        return float(r[0]), float(r[1])

    def output(self):
        """The scaled stem as (N, C), or None when measuring only; checks that nothing around it was written."""
        if self.mode == "none":
            assert torch.equal(self.buf[self.off:self.off + self.n].cpu(),
                               torch.from_numpy(np.ascontiguousarray(self.dense_input())))
            return None
        b = (self.obuf if self.mode == "sep" else self.buf).cpu().numpy()
        assert np.all(np.isnan(b[:self.off])) and np.all(np.isnan(b[self.off + self.n:]))
        flat = b[self.off:self.off + self.n]
        return flat.reshape(self.C, self.N).T if self.layout == "cn" else flat.reshape(self.N, self.C)

    def dense_input(self):
        return self.x.T.reshape(-1) if self.layout == "cn" else self.x.reshape(-1)


def _stem_shape(s):
    return (s.rirs.shape[1] if hasattr(s, "rirs") else s.rir.shape[0]), s.dry.shape[0]


def _scene(rng, n_sources=12):
    """Moving, static and long-RIR sources with C = 1..8 and different N; some without targets, one with a direct
    target.  Returns (sources, targets, direct index)."""
    from sonicsim_b200 import render
    srcs, targets = [], []
    for i in range(n_sources):
        C = 1 + i % 8
        N = int(rng.integers(20000, 70000)) if i != 5 else 5000              # one clip shorter than a gating block
        kind = i % 3
        L = int(rng.integers(4097, 9000)) if kind == 2 else int(rng.integers(200, 3000))
        x = so.synth_dry(rng, N)
        if kind == 0:
            srcs.append(render.StaticSource(x, so.synth_rirs(rng, 1, C, L)[0]))
        else:
            P = int(rng.integers(3, 9))
            pos = so.synth_path(rng, P)
            np.random.seed(i)
            srcs.append(render.MovingSource(x, so.synth_rirs(rng, P, C, L), render.trajectory_bounds(pos, N)))
        targets.append(None if i in (2, 7, 10) else float(rng.uniform(-33, -15)))
    direct = 4
    srcs[direct] = srcs[direct]._replace(direct_taps=40)
    return srcs, targets, direct

MALFORMED = {"blk_lo NULL": ("blk_lo", None), "blk_hi NULL": ("blk_hi", None), "n_e 0": ("n_e", 0),
             "n_blocks -1": ("n_blocks", -1), "rate 0": ("rate", 0.0), "rate NaN": ("rate", NAN),
             "block_size 0": ("block_size", 0.0), "block_size NaN": ("block_size", NAN)}
