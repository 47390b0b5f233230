"""Generate tests/golden/crop_draw.npz: the crop starts the separation dataloader's start loop chooses
(/root/reference/separation/look2hear/datas/movingdatamodule.py:81-99, with compute_mch_rms_dB of :29-32), executed
verbatim on seeded synthetic float32 `speaker_wav` with silent stretches.  Run in the authoring container only:

    python oracle/make_crop_draw_golden.py

`random` is a stub whose randint(a, b) returns a + floor(u * (b - a + 1)) from a given list of u, so that the same u
drive tests/draw_reference.py, the CPU emulation of k_draw and the device.  The fixture holds the inputs and the
reference's starts, so the tests that read it need neither /root/reference nor this script.  TEST INFRASTRUCTURE.
"""
import math
import os
import sys
import textwrap

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import draw_reference as dr                         # noqa: E402

SRC = "/root/reference/separation/look2hear/datas/movingdatamodule.py"
OUT = os.path.join(ROOT, "tests", "golden", "crop_draw.npz")
RATE, DURATION = 100, 4.0                           # a crop of 400 samples
LEN = int(RATE * DURATION)
TRIES = 101


def reference_lines():
    lines = open(SRC).read().split("\n")
    rms = "\n".join(lines[28:32])                   # :29-32
    loop = textwrap.dedent("\n".join(lines[80:99]))  # :81-99
    assert rms.startswith("def compute_mch_rms_dB") and loop.startswith("start = 0"), (rms, loop)
    assert "break" in loop.split("\n")[-1]
    return rms, loop


class StubRandom:
    def __init__(self, u):
        self.u, self.calls = list(u), 0

    def randint(self, a, b):
        v = self.u[self.calls]
        self.calls += 1
        return int(a + math.floor(v * (b - a + 1)))


class Self:
    sample_rate, duration = RATE, DURATION

    def __init__(self, S):
        self.num_spks = S


def run_reference(wav, u):
    import torch
    rms, loop = reference_lines()
    ns = {"torch": torch, "np": np}
    exec(rms, ns)
    ns.update(self=Self(wav.shape[0]), speaker_wav=torch.from_numpy(wav.copy()), random=StubRandom(u))
    exec(loop, ns)
    used = ns["for_idx"] + 1 if ns["for_idx"] <= TRIES - 1 else 0
    assert ns["random"].calls == (used if used else TRIES)
    return int(ns["start"]), used


def u_for(starts, M):
    return np.array([(s + 0.5) / M for s in starts], np.float64)


def loud(rng, shape):
    return (0.1 * rng.standard_normal(shape)).astype(np.float32)


def cases():
    rng = np.random.default_rng(2026)
    T = 3000
    M = T - LEN + 1
    out = []
    # S = 1, mono: the first try passes
    w = loud(rng, (1, T)); w[0, :1000] = 0
    out.append(("first_try", w, u_for([1500] + [0] * 100, M)))
    # S = 2: speaker 1 is loud only in [2000, 2600): the first 100 tries land before it, only try 100 passes
    w = loud(rng, (2, T)); w[1, :2000] = 0; w[1, 2600:] = 0
    out.append(("only_try_100", w, u_for(list(rng.integers(0, 1500, 100)) + [2100], M)))
    # S = 3: speaker 2 is silent wherever the tries land: every try silent, the last start is kept
    w = loud(rng, (3, T)); w[2, :2400] = 0
    out.append(("all_silent", w, u_for(list(rng.integers(0, 1900, TRIES)), M)))
    # S = 2 with channels, (S, C, T): gaps in both speakers, random tries
    w = loud(rng, (2, 3, T)); w[0, :, 300:1400] = 0; w[1, :, 1800:2900] = 0
    out.append(("channels", w, rng.random(TRIES)))
    # S = 3, mono, dataloader-like gaps of several lengths, random tries, some silent before a pass
    for j in range(4):
        w = loud(rng, (3, T))
        for s in range(3):
            a = int(rng.integers(0, T - 900)); w[s, a:a + int(rng.integers(400, 900))] = 0
        out.append(("gaps%d" % j, w, rng.random(TRIES)))
    return out


def main():
    data = {}
    names = []
    for k, (name, wav, u) in enumerate(cases()):
        start, used = run_reference(wav, u)
        mono = wav.ndim == 2
        tabs = [dr.level_table(wav[s][None] if mono else wav[s], mono) for s in range(wav.shape[0])]
        D = [LEN if mono else wav.shape[1] * LEN] * wav.shape[0]
        assert dr.draw(tabs, D, [wav.shape[-1]] * wav.shape[0], LEN, u) == (start, used), name
        assert dr.margins(tabs, D, [wav.shape[-1]] * wav.shape[0], LEN, u) > 1e-3, name
        data["wav%d" % k], data["u%d" % k] = wav, u
        data["start%d" % k], data["used%d" % k] = np.int64(start), np.int64(used)
        names.append(name)
        print(name, "S=%d" % wav.shape[0], "start", start, "used", used)
    data["names"] = np.array(names)
    data["len"] = np.int64(LEN)
    data["n_cases"] = np.int64(len(names))
    np.savez_compressed(OUT, **data)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
