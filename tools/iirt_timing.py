"""Time iirt on the GPU: clips of 10 s at 22 050 Hz, resident on the device, librosa's defaults
(res_type="polyphase").  Prints the card name and power limit, then for 1 024 clips and for one clip the time per
call (CUDA events recorded on the library's stream before and after each call, after warm-up; least and median of
the repeats), the launches per call, and the FP64 and scratch-traffic shares computed from shapes against the
H100 SXM's FP64 issue rate (64 results per clock per SM, 132 SMs at 1.98 GHz: 1.67e13 instructions/s; the filter
issues no FMA) and its 3.35 TB/s of HBM3.  ``--profile`` instead runs torch.profiler once and splits the device
time by kernel.

    python tools/iirt_timing.py [--clips 1024] [--seconds 10] [--reps 5] [--profile]
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import librosa_b200 as lb  # noqa: E402
from librosa_b200.core import semitone as S  # noqa: E402

FP64_RATE = 64 * 132 * 1.98e9   # FP64 instructions per second
HBM = 3.35e12                   # bytes per second


def card() -> str:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def work(p: S.Plan, clips: int):
    """(FP64 instructions of the two filter passes, float64 scratch bytes moved) for ``clips`` clips: 9 per sample
    and section (5 multiplies, 4 adds) over n + 2 padlen forward and n + padlen backward samples; the scratch is
    written forward (n + padlen rows), read and rewritten backward, and read once by the STMSP."""
    instr = traffic = 0
    for b, (ns, pl) in enumerate(p.bank.info):
        n = p.rates[p.bank.rate_of[b]].n
        instr += 9 * int(ns) * ((n + 2 * int(pl)) + (n + int(pl)))
        traffic += 8 * ((n + pl) + (n + pl) + n + n)
    return instr * clips, int(traffic) * clips


def timed(y, reps, kw):
    ctx = lb.default_context()
    for _ in range(2):
        lb.iirt(y, **kw).free()
    ctx.synchronize()
    times = []
    for _ in range(reps):
        e0 = ctx.event().record()
        out = lb.iirt(y, **kw)
        e1 = ctx.event().record()
        ctx.synchronize()
        times.append(e0.elapsed_ms(e1) / 1e3)
        shape = out.shape
        out.free()
    before = ctx.launch_count
    lb.iirt(y, **kw).free()
    return times, shape, ctx.launch_count - before


def family(name: str) -> str:
    for key in ("sosfiltfilt", "stmsp", "resample_poly", "pad_center"):
        if key in name:
            return key
    return name[:40]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    sr = 22050
    n = int(a.seconds * sr)
    kw = dict(sr=sr, res_type="polyphase")
    print(f"card: {card()}")
    y = (0.1 * np.random.default_rng(0).standard_normal((a.clips, n))).astype(np.float32)
    dy = lb.to_device(y)
    if a.profile:
        import torch
        from torch.profiler import ProfilerActivity, profile

        lb.iirt(dy, **kw).free()
        lb.default_context().synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            lb.iirt(dy, **kw).free()
            lb.default_context().synchronize()
        fam = {}
        for ev in prof.key_averages():
            t = getattr(ev, "device_time_total", None) or getattr(ev, "cuda_time_total", 0)
            if t and ev.key and "Memcpy" not in ev.key and "Memset" not in ev.key:
                tot, cnt = fam.get(family(ev.key), (0.0, 0))
                fam[family(ev.key)] = (tot + t, cnt + ev.count)
        for f, (tot, cnt) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
            print(f"  {f:16s} {tot / 1e3:9.3f} ms  ({cnt} launches)")
        del torch
        return
    p = S.plan((a.clips, n), sr=sr, win_length=2048, hop_length=None, center=True, tuning=0.0, pad_mode="constant",
               res_type="polyphase", kwargs={})
    for clips, x in ((a.clips, dy), (1, lb.to_device(y[:1]))):
        times, shape, launches = timed(x, a.reps, kw)
        instr, traffic = work(p, clips)
        t = min(times)
        print(f"iirt {clips} x {a.seconds:g} s -> {shape}: CUDA events around the call: least {t * 1e3:.2f} ms, "
              f"median {float(np.median(times)) * 1e3:.2f} ms over {a.reps} calls; {launches} launches; "
              f"{instr:.3g} FP64 instructions -> {instr / FP64_RATE * 1e3:.2f} ms at the issue rate "
              f"({instr / FP64_RATE / t:.1%} of the call); {traffic / 1e9:.1f} GB of scratch -> "
              f"{traffic / HBM * 1e3:.2f} ms at 3.35 TB/s ({traffic / HBM / t:.1%} of the call)")
        x.free()


if __name__ == "__main__":
    main()
