"""Device-resident render time of the BASELINE.json configs (informational; bench.py's line is configs[1])."""
import sys, os, subprocess
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import sonicsim_oracle as so
from sonicsim_b200 import render

R = render.Renderer(0)
dev = torch.device("cuda", 0)


def card():
    """Name and power limit of cuda:0 (the numbers below depend on both)."""
    props = torch.cuda.get_device_properties(0)
    limit = "unknown"
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=uuid,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        uuid = str(getattr(props, "uuid", ""))
        rows = [r.split(", ") for r in q if r]
        match = [r for r in rows if uuid and uuid in r[0]] or rows[:1]
        if match:
            limit = match[0][1]
    except (OSError, subprocess.SubprocessError):
        pass
    return "%s, power limit %s" % (props.name, limit)


print("device:", card())


def moving(rng, N, P, C, L, sr=16000, t60=0.5):
    x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L, sr=sr, t60=t60), so.synth_path(rng, P)
    b = render.trajectory_bounds(pos, N)
    return render.MovingSource(torch.from_numpy(x).to(dev), torch.from_numpy(h).to(dev), torch.from_numpy(b).to(dev), b), \
        torch.empty((C, N), device=dev)


def static(rng, N, C, L):
    x, h = so.synth_dry(rng, N), so.synth_rirs(rng, 1, C, L)[0]
    return render.StaticSource(torch.from_numpy(x).to(dev), torch.from_numpy(h).to(dev)), torch.empty((C, N), device=dev)


def timeit(name, srcs, outs, audio_s, reps=10):
    for _ in range(3):
        R.render_device(srcs, outs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        R.render_device(srcs, outs)
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    print("%-58s %9.3f ms  %12.0f audio-s/s" % (name, ms, audio_s / (ms / 1e3)))


rng = np.random.default_rng(0)
np.random.seed(0)
s, o = static(rng, 64000, 1, 4096)
timeit("cfg1: 1 static, mono, L=4096, 4 s (single call)", [s], [o], 4.0, 50)
pairs = [moving(rng, 480000, 40, 6, 4096) for _ in range(2)]
timeit("cfg2: 2 spk, 6 mic, 40 pt, 30 s (single utterance)", [p[0] for p in pairs], [p[1] for p in pairs], 30.0, 20)
items = []
for _ in range(8):
    items += [moving(rng, 960000, 60, 6, 4096) for _ in range(2)] + [static(rng, 960000, 6, 4096) for _ in range(2)]
timeit("cfg3: 8 utt x (2 moving 60 pt + 2 static), 6 mic, 60 s", [p[0] for p in items], [p[1] for p in items], 8 * 60.0, 5)
trip = [moving(rng, 2880000, 120, 4, 32768, sr=48000, t60=1.5) for _ in range(3)]
timeit("cfg4: 3 moving, 4 ch, 120 pt, L=32768, 60 s @48k", [p[0] for p in trip], [p[1] for p in trip], 60.0, 3)


# cfg5: the speaker's direct-path target (every RIR row cut 2.5 ms = 40 taps after its peak) rendered two ways, timed
# call by call in alternating order: (a) as a second moving source whose RIRs were truncated on the host, (b) as the
# SS_DIRECT_TARGET stem of the speaker itself (dry-window transforms and X staging shared with the reverberant stem).
# Once for one utterance (a single call is mostly launch latency) and once for a batch of 8.
def cfg5_forms(n_utt, N=960000, P=40, C=2, L=4096, taps=40):
    g = lambda a: torch.from_numpy(a).to(dev)
    fa = dict(sources=[], outs=[])
    fb = dict(sources=[], outs=[], direct_outs=[])
    pairs = []
    for _ in range(n_utt):
        x, h, pos = so.synth_dry(rng, N), so.synth_rirs(rng, P, C, L), so.synth_path(rng, P)
        cut = np.minimum(L, np.abs(h).argmax(axis=-1) + taps)
        hd = np.where(np.arange(L) < cut[..., None], h, np.float32(0)).astype(np.float32)
        b = render.trajectory_bounds(pos, N)
        spk = render.MovingSource(g(x), g(h), g(b), b)
        noise, music = static(rng, N, C, L), static(rng, N, C, L)
        o_rev, o_a, o_b = (torch.empty((C, N), device=dev) for _ in range(3))
        fa["sources"] += [spk, render.MovingSource(g(x), g(hd), g(b), b), noise[0], music[0]]
        fa["outs"] += [o_rev, o_a, noise[1], music[1]]
        fb["sources"] += [spk._replace(direct_taps=taps), noise[0], music[0]]
        fb["outs"] += [o_rev, noise[1], music[1]]
        fb["direct_outs"] += [o_b, None, None]
        pairs.append((o_a, o_b))
    return fa, fb, pairs


def alternate(n_utt, reps=40):
    fa, fb, pairs = cfg5_forms(n_utt)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = {"a": [], "b": []}
    for _ in range(3):
        R.render_device(**fa); R.render_device(**fb)
    for rep in range(reps):
        for k in ("ab" if rep % 2 == 0 else "ba"):
            torch.cuda.synchronize()
            e0.record()
            R.render_device(**(fa if k == "a" else fb))
            e1.record(); torch.cuda.synchronize()
            ms[k].append(e0.elapsed_time(e1))
    same = all(torch.equal(a, b) for a, b in pairs)
    for k, name in (("a", "direct set as a 2nd moving source"), ("b", "direct target of the speaker (one source)")):
        med = float(np.median(ms[k]))
        print("cfg5 x%d utt: %-44s %9.3f ms  %12.0f audio-s/s  (median of %d, min %.3f)"
              % (n_utt, name, med, n_utt * 60.0 / (med / 1e3), len(ms[k]), min(ms[k])))
    print("cfg5 x%d utt: direct stems of the two forms bit-identical: %s;  time b / a = %.3f"
          % (n_utt, same, np.median(ms["b"]) / np.median(ms["a"])))


alternate(1)
alternate(8, reps=20)
