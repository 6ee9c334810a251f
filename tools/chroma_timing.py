"""Time the constant-Q chroma features on the GPU: 1024 clips of 10 s at 22 050 Hz, resident on the device,
chroma_cqt(y=..., res_type="polyphase") at librosa's defaults (252 bins, 36 per octave), then chroma_cens and
tonnetz on the same input.  Prints the card name and power limit, the time per call (CUDA events recorded on the
library's stream before and after each call, after warm-up; least and median of the repeats), the launches per
call, the device time per kernel family from one torch.profiler run of its own (STFT, resample, projection,
fold, smooth), and the fold's share of the time its bytes need at the data-sheet 3.35 TB/s.

    python tools/chroma_timing.py [--clips 1024] [--seconds 10] [--reps 10]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import librosa_b200 as lb  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def family(name: str) -> str:
    for key, fam in (("chroma_fold", "fold"), ("chroma_smooth", "smooth"), ("cqt_project", "projection"),
                     ("resample_poly", "resample"), ("finite_scan", "finite scan"), ("pip", "tuning"),
                     ("tuning", "tuning")):
        if key in name:
            return fam
    return "stft"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    sr = 22050
    y = np.random.default_rng(0).standard_normal((a.clips, int(a.seconds * sr))).astype(np.float32)
    ctx = lb.default_context()
    dy = lb.to_device(y)
    F = lb.feature
    calls = {"chroma_cqt": lambda: F.chroma_cqt(y=dy, sr=sr, res_type="polyphase"),
             "chroma_cens": lambda: F.chroma_cens(y=dy, sr=sr, res_type="polyphase"),
             "tonnetz": lambda: F.tonnetz(y=dy, sr=sr, res_type="polyphase"),
             "cqt (252 bins, tuning=None)": lambda: lb.cqt(dy, sr=sr, n_bins=252, bins_per_octave=36, tuning=None,
                                                           res_type="polyphase")}
    print(f"card: {card()}")
    for name, fn in calls.items():
        for _ in range(3):
            fn().free()
        ctx.synchronize()
        times = []
        for _ in range(a.reps):
            e0 = ctx.event().record()
            out = fn()
            e1 = ctx.event().record()
            ctx.synchronize()
            times.append(e0.elapsed_ms(e1))
            shape = out.shape
            out.free()
        l0 = ctx.launch_count
        fn().free()
        print(f"{name} {a.clips} x {a.seconds:g} s -> {shape}: CUDA events around the call: least {min(times):.2f} ms, "
              f"median {float(np.median(times)):.2f} ms over {a.reps} calls; {ctx.launch_count - l0} launches per call")

    import torch
    from torch.profiler import ProfilerActivity, profile

    T = 1 + int(a.seconds * sr) // 512
    fold_bytes = a.clips * T * (252 * 8 + 12 * 4)
    for name in ("chroma_cqt", "chroma_cens"):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(3):
                calls[name]().free()
            ctx.synchronize()
        fam = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if t and ev.key and "Memcpy" not in ev.key and "Memset" not in ev.key:
                f = family(ev.key)
                tot, cnt = fam.get(f, (0.0, 0))
                fam[f] = (tot + t, cnt + ev.count)
        print(f"{name}: device time per kernel family (torch.profiler)")
        for f, (tot, cnt) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
            print(f"  {f:12s} {tot / 3 / 1e3:8.3f} ms per call  ({cnt // 3} launches per call)")
        if name == "chroma_cqt" and "fold" in fam:
            ms = fam["fold"][0] / 3 / 1e3
            bound = fold_bytes / HBM_BYTES_PER_S * 1e3
            print(f"  fold: {fold_bytes / 1e9:.3f} GB read and written; {bound:.3f} ms at 3.35 TB/s; "
                  f"{bound / ms * 100:.0f} % of that bound")
    del torch
    dy.free()


if __name__ == "__main__":
    main()
