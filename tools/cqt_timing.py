"""Time cqt, hybrid_cqt or pseudo_cqt on the GPU: 1024 clips of 10 s at 22 050 Hz, resident on the device,
librosa's defaults (res_type="polyphase"; pseudo_cqt from C2 with 72 bins, since its defaults need n_fft=16384).
Prints the card name and power limit, the time per call (CUDA events recorded on the library's stream before and
after each call, after warm-up; least and median of the repeats; the host clock to the end of a synchronise beside
it), and the device time per kernel family from one torch.profiler run of its own (STFTs, resamples, projection).
With --fn hybrid_cqt or pseudo_cqt, cqt at the same settings is timed in the same loop, the two calls alternating.

    python tools/cqt_timing.py [--fn cqt|hybrid_cqt|pseudo_cqt] [--clips 1024] [--seconds 10] [--reps 10]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import librosa_b200 as lb  # noqa: E402


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def family(name: str) -> str:
    if "cqt_project" in name:
        return "projection"
    if "resample_poly" in name:
        return "resample"
    if "finite_scan" in name:
        return "finite scan"
    return "stft"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--fn", choices=("cqt", "hybrid_cqt", "pseudo_cqt"), default="cqt")
    ap.add_argument("--clips", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    sr = 22050
    y = np.random.default_rng(0).standard_normal((a.clips, int(a.seconds * sr))).astype(np.float32)
    ctx = lb.default_context()
    dy = lb.to_device(y)
    kw = dict(sr=sr, res_type="polyphase")
    calls = {"cqt": lambda: lb.cqt(dy, **kw)}
    if a.fn == "hybrid_cqt":
        calls[a.fn] = lambda: lb.hybrid_cqt(dy, **kw)
    elif a.fn == "pseudo_cqt":
        pkw = dict(sr=sr, fmin=65.40639132514966, n_bins=72)   # C2
        calls = {"cqt": lambda: lb.cqt(dy, **kw, **{k: v for k, v in pkw.items() if k != "sr"}),
                 a.fn: lambda: lb.pseudo_cqt(dy, **pkw)}
    for _ in range(3):
        for fn in calls.values():
            fn().free()
    ctx.synchronize()
    times = {k: [] for k in calls}
    walls = {k: [] for k in calls}
    shapes, launches = {}, {}
    for _ in range(a.reps):
        for name, fn in calls.items():   # alternating, so both see the same conditions
            t0 = time.perf_counter()
            e0 = ctx.event().record()
            C = fn()
            e1 = ctx.event().record()
            ctx.synchronize()
            walls[name].append(time.perf_counter() - t0)
            times[name].append(e0.elapsed_ms(e1) / 1e3)
            shapes[name] = C.shape
            C.free()
    for name, fn in calls.items():
        launches0 = ctx.launch_count
        fn().free()
        launches[name] = ctx.launch_count - launches0
    print(f"card: {card()}")
    for name in calls:
        t, w = times[name], walls[name]
        print(f"{name} {a.clips} x {a.seconds:g} s -> {shapes[name]}: CUDA events around the call: least "
              f"{min(t) * 1e3:.2f} ms, median {float(np.median(t)) * 1e3:.2f} ms per call over {a.reps} calls; host "
              f"clock to the end of a synchronise: median {float(np.median(w)) * 1e3:.2f} ms; {launches[name]} "
              "launches per call")

    import torch
    from torch.profiler import ProfilerActivity, profile

    fn = calls[a.fn]
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(3):
            fn().free()
        ctx.synchronize()
    fam = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
        if t and ev.key and "Memcpy" not in ev.key and "Memset" not in ev.key:
            f = family(ev.key)
            tot, cnt = fam.get(f, (0.0, 0))
            fam[f] = (tot + t, cnt + ev.count)
    print(f"{a.fn} per kernel family (torch.profiler):")
    for f, (tot, cnt) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
        print(f"  {f:12s} {tot / 3 / 1e3:8.3f} ms per call  ({cnt // 3} launches per call)")
    del torch
    dy.free()


if __name__ == "__main__":
    main()
