"""REPET-SIM timing: decompose.nn_filter(|stft|, aggregate=np.median, metric="cosine", width=86) of a synthetic 5-minute
22 050 Hz signal (n_fft 2048, hop 512: 1 025 bins x 12 920 frames, float32, on the device), with CUDA events around
`reps` calls after warm-up, and the time of each kernel from torch.profiler in a separate pass.  Next to them, the
least times from the shapes: the FP64 Gram product (2 t^2 d FLOP, both triangles, at the data sheet's 67 TFLOP/s FP64
tensor-core rate) and the bytes the distance workspace, the selection and the aggregation must move at 3.35 TB/s.
``card`` is the GPU's name, power limit and maximum SM clock, read in the same run.  ``oracle_cpu_s`` is the NumPy
oracle (tests/nn_filter_oracle.py) on the same input: its graph and its aggregation over the GPU's graph.

    python tools/nn_filter_timing.py [seconds=300] [reps=3] [oracle=1] > nn_filter_timing.json
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np

import librosa_b200 as lb

seconds = float(sys.argv[1]) if len(sys.argv) > 1 else 300.0
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 3
with_oracle = (sys.argv[3] != "0") if len(sys.argv) > 3 else True
sr, width = 22050, 86
ctx = lb.default_context()

# a repeating accompaniment (four chords of harmonic tones, period 8 s) under a non-repeating voice-like melody
rng = np.random.default_rng(0)
n = int(seconds * sr)
tt = np.arange(n) / sr
y = np.zeros(n)
for c, f0 in enumerate((110.0, 146.8, 164.8, 130.8)):
    on = ((tt // 2.0) % 4) == c
    for h in range(1, 6):
        y += on * 0.1 / h * np.sin(2 * np.pi * f0 * h * tt)
y += 0.05 * np.sin(2 * np.pi * (300 + 100 * np.sin(2 * np.pi * 0.13 * tt)) * tt)
y += 0.01 * rng.standard_normal(n)
dy = ctx.to_device(y.astype(np.float32))
S = lb.core.spectrum._spectrogram(y=dy, n_fft=2048, hop_length=512, power=1)[0]
dy.free()
F, t = S.shape
kw = dict(aggregate=np.median, metric="cosine", width=width)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[ctx.device] if q.returncode == 0 else "unknown"


out = {"S_shape": [F, t], "S_layout": S.layout, "width": width, "reps": reps, "card": card()}
res = lb.decompose.nn_filter(S, **kw)   # warm-up
res.free()
ctx.synchronize()
e0, e1 = ctx.event(), ctx.event()
l0 = ctx.launch_count
e0.record()
for _ in range(reps):
    lb.decompose.nn_filter(S, **kw).free()
e1.record()
ctx.synchronize()
out["nn_filter_ms"] = round(e0.elapsed_ms(e1) / reps, 2)
out["launches_per_call"] = (ctx.launch_count - l0) / reps
k = int(2 * np.ceil(np.sqrt(t - 2 * width + 1)))
M = min(t - 1, k + 2 * width)
flop = 2.0 * t * t * F
moved = 2 * 8.0 * t * t + 8.0 * t * t * 8 + 4.0 * F * t * (k + 1)   # workspace written + read (8 radix passes)
out["k"], out["candidates"] = k, M
out["bounds"] = {"gram_fp64_flop": flop, "gram_us_at_67_tflops": round(flop / 67e12 * 1e6, 1),
                 "bytes": moved, "bytes_us_at_3.35_tbs": round(moved / 3.35e12 * 1e6, 1)}

import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

with profile(activities=[ProfilerActivity.CUDA]) as prof:
    lb.decompose.nn_filter(S, **kw).free()
    ctx.synchronize()
kern = {}
for ev in prof.key_averages():
    if "nn_" in ev.key or "transpose" in ev.key:
        kern[ev.key[:80]] = {"calls": ev.count, "total_ms": round(ev.device_time_total / 1e3, 3)}
out["kernels"] = kern

if with_oracle:
    import nn_filter_oracle as NO

    Sh = S.get()
    t0 = time.perf_counter()
    rec, _ = NO.graph(Sh, metric="cosine", width=width)
    out["oracle_cpu_graph_s"] = round(time.perf_counter() - t0, 1)
    gpu_rec = lb.segment.recurrence_matrix(Sh, metric="cosine", width=width, sparse=True)
    t0 = time.perf_counter()
    want = NO.aggregate(Sh, gpu_rec, np.median)
    out["oracle_cpu_median_s"] = round(time.perf_counter() - t0, 1)
    got = lb.decompose.nn_filter(Sh, **kw)
    out["bit_identical_to_oracle_aggregation"] = bool(np.array_equal(np.ascontiguousarray(got).view(np.uint8),
                                                                     np.ascontiguousarray(want).view(np.uint8)))
    out["graph_columns_equal_to_oracle"] = int(sum(
        np.array_equal(rec.indices[rec.indptr[i]:rec.indptr[i + 1]], gpu_rec.indices[gpu_rec.indptr[i]:gpu_rec.indptr[i + 1]])
        for i in range(t)))
print(json.dumps(out))
