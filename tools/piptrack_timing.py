"""Device-resident timings of piptrack, pitch_tuning and util.localmax on |stft| of a batch of 10 s clips at 22 050 Hz
(n_fft 2048, hop 512: 1 025 bins x 431 frames per clip, "ft" layout; bench.py's cfg2 signals), with CUDA events around
`reps` calls after warm-up, next to each call's least time from the shapes: the bytes it must read and write at
3.35 TB/s (data sheet of the H100 SXM).  ``card`` is the GPU's name, power limit and maximum SM clock, read in the
same run.

piptrack(S=device) is two launches: a pass that decides the reference's S.min() < 0 (it reads S once more) and the
tracking kernel.  ``kernels`` also times the tracking kernel alone through the C ABI, as piptrack(S=host) or
piptrack(y=...) launch it (no sign pass).

    python tools/piptrack_timing.py [clips=1024] [reps=20] > piptrack_timing.json
"""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np

import bench
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200.core import pitch as P

clips = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
ctx = lb.default_context()
dev = ctx.to_device(bench.make_batch(dict(bench.WORKLOADS["cfg2"], clips=clips), 0))
S, n_fft = lb.core.spectrum._spectrogram(y=dev, n_fft=2048, hop_length=512, power=1)
dev.free()
nbytes = S.nbytes
pitches, mags = lb.piptrack(S=S, sr=22050)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[ctx.device] if q.returncode == 0 else "unknown"


def timed(call, moved, free=True):
    for _ in range(3):
        r = call()
        if free:
            for d in (r if isinstance(r, tuple) else (r,)):
                d.free()
    ctx.synchronize()
    e0, e1 = ctx.event(), ctx.event()
    l0 = ctx.launch_count
    e0.record()
    for _ in range(reps):
        r = call()
        if free:
            for d in (r if isinstance(r, tuple) else (r,)):
                d.free()
    e1.record()
    ctx.synchronize()
    us = e0.elapsed_ms(e1) / reps * 1e3
    bound_us = moved / 3.35e12 * 1e6
    return {"us_per_call": round(us, 1), "bytes": int(moved), "bound_us": round(bound_us, 1),
            "share_of_bound": round(bound_us / us, 3), "launches_per_call": (ctx.launch_count - l0) / reps}


CALLS = {   # name: (call, bytes read + written, returns device arrays)
    "piptrack(S=device)": (lambda: lb.piptrack(S=S, sr=22050), 2 * nbytes + 2 * nbytes, True),
    "pitch_tuning(pitches)": (lambda: lb.pitch_tuning(pitches), nbytes, False),
    "util.localmax(S, axis=-2)": (lambda: lb.util.localmax(S, axis=-2), nbytes + nbytes // 4, True),
}
out = {"clips": clips, "S_shape": list(S.shape), "S_layout": S.layout, "reps": reps, "card": card(),
       "peaks": int(np.count_nonzero(np.asarray(pitches.get()))), "calls": {}}
for name, (call, moved, free) in CALLS.items():
    out["calls"][name] = timed(call, moved, free)
    print(name, out["calls"][name], file=sys.stderr)

desc = P._piptrack_desc(S.shape[-2], n_fft, np.dtype(np.float32), sr=22050, fmin=150.0, fmax=4000.0, threshold=0.1,
                        ref=None)
desc.abs_mode, desc.layout_c = 0, 0
kernel = lambda: nat.check(nat.lib().b2l_piptrack(ctx.handle, C.byref(desc), C.c_void_p(S.ptr), S.shape[0],
                                                  S.shape[-2], S.shape[-1], C.c_void_p(pitches.ptr),
                                                  C.c_void_p(mags.ptr)))
out["kernels"] = {"piptrack_kernel (no sign pass)": timed(kernel, 3 * nbytes, False)}
print(out["kernels"], file=sys.stderr)
print(json.dumps(out))
