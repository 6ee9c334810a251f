"""Device-resident timings of feature.delta and feature.stack_memory on the MFCCs of a batch of 10 s clips at 22 050 Hz
(20 x 431 per clip; bench.py's cfg2 batch), with CUDA events around `reps` calls after warm-up, next to each call's
least time from the shapes: the bytes it must read and write at 3.35 TB/s (data sheet of the H100 SXM).  ``card`` is
the GPU's name, power limit and maximum SM clock, read in the same run.

delta's default mode="interp" reads the status word after its launch (SciPy raises on non-finite edge windows), so its
calls wait for the device; mode="nearest" makes the same launch without that read.  A public call also spends host
time (argument checks, staging, result allocation) that can exceed the kernel's, so ``kernels`` times the C-ABI
launches alone, back to back into one output, with the tables of the public call.

    python tools/featutil_timing.py [clips=1024] [reps=50] > featutil_timing.json
"""
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench
import librosa_b200 as lb
from librosa_b200 import _native as nat
from librosa_b200 import _pipeline as pl
from librosa_b200.feature import utils as U

clips = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 50
ctx = lb.default_context()
dev = ctx.to_device(bench.make_batch(dict(bench.WORKLOADS["cfg2"], clips=clips), 0))
M = lb.feature.mfcc(y=dev, sr=22050)
dev.free()
nbytes = M.nbytes


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[ctx.device] if q.returncode == 0 else "unknown"


CALLS = {   # name: (call, bytes read + written)
    "delta(order=1)": (lambda: lb.feature.delta(M), 2 * nbytes),
    "delta(order=2)": (lambda: lb.feature.delta(M, order=2), 2 * nbytes),
    "delta(order=1, mode=nearest)": (lambda: lb.feature.delta(M, mode="nearest"), 2 * nbytes),
    "delta(order=2, mode=nearest)": (lambda: lb.feature.delta(M, order=2, mode="nearest"), 2 * nbytes),
    "stack_memory(n_steps=3)": (lambda: lb.feature.stack_memory(M, n_steps=3), 4 * nbytes),
}

out = {"clips": clips, "mfcc_shape": list(M.shape), "mfcc_layout": M.layout, "reps": reps, "card": card(), "calls": {}}
for name, (call, moved) in CALLS.items():
    for _ in range(5):
        call().free()
    ctx.synchronize()
    e0, e1 = ctx.event(), ctx.event()
    l0 = ctx.launch_count
    e0.record()
    for _ in range(reps):
        call().free()
    e1.record()
    ctx.synchronize()
    us = e0.elapsed_ms(e1) / reps * 1e3
    bound_us = moved / 3.35e12 * 1e6
    out["calls"][name] = {"us_per_call": round(us, 1), "bytes": moved, "bound_us": round(bound_us, 1),
                          "share_of_bound": round(bound_us / us, 3), "launches_per_call": (ctx.launch_count - l0) / reps}
    print(name, out["calls"][name], file=sys.stderr)


def delta_launch(order, mode):
    fw, sym, key = U._taps(9, order, order, 1.0)
    pad, pad_key = U._pad_table(M.shape[-1], 4, 4, U._NDIMAGE_PAD[mode])
    desc = nat.DeltaDesc(width=9, sym=sym, interp=int(mode == "interp"), f64=0, cval=0.0)
    desc.d_taps = pl.f64_constant(ctx, ("delta_taps", key), fw)
    desc.d_pad = pl.f64_constant(ctx, ("delta_pad", pad_key), pad)
    E, e_key = U._edge_table(9, order, order, 1.0)
    desc.d_edge = pl.f64_constant(ctx, ("delta_edge", e_key), E)
    y = ctx.empty(M.shape, M.dtype)
    rows = pl.clip_count(M.shape[:-1])
    return lambda: nat.check(nat.lib().b2l_delta(ctx.handle, C.byref(desc), C.c_void_p(M.ptr), rows, M.shape[-1], 1,
                                                 C.c_void_p(y.ptr))), y


def stack_launch(n_steps):
    table = U.pad_index_table(M.shape[-1], n_steps - 1, 0, "constant")
    desc = nat.StackDesc(elem_size=4, n_steps=n_steps, delay=1, clip_stride=M.shape[-2] * M.shape[-1],
                         row_stride=M.shape[-1], col_stride=1)
    d_pad = pl.f64_constant(ctx, ("stack_pad", pl.digest(table)), table)
    y = ctx.empty(M.shape[:-2] + (n_steps * M.shape[-2], M.shape[-1]), M.dtype)
    return lambda: nat.check(nat.lib().b2l_stack_memory(ctx.handle, C.byref(desc), C.c_void_p(M.ptr), M.shape[0],
                                                        M.shape[-2], M.shape[-1], C.c_void_p(d_pad),
                                                        C.c_void_p(y.ptr))), y


out["kernels"] = {}
for name, (make, moved) in {"delta_rows_kernel(order=1, interp)": (lambda: delta_launch(1, "interp"), 2 * nbytes),
                            "delta_rows_kernel(order=2, interp)": (lambda: delta_launch(2, "interp"), 2 * nbytes),
                            "delta_rows_kernel(order=1, nearest)": (lambda: delta_launch(1, "nearest"), 2 * nbytes),
                            "stack_memory_kernel(n_steps=3)": (lambda: stack_launch(3), 4 * nbytes)}.items():
    launch, y = make()
    for _ in range(5):
        launch()
    ctx.synchronize()
    e0, e1 = ctx.event(), ctx.event()
    e0.record()
    for _ in range(reps):
        launch()
    e1.record()
    ctx.synchronize()
    us = e0.elapsed_ms(e1) / reps * 1e3
    bound_us = moved / 3.35e12 * 1e6
    out["kernels"][name] = {"us": round(us, 1), "bound_us": round(bound_us, 1), "share_of_bound": round(bound_us / us, 3)}
    print(name, out["kernels"][name], file=sys.stderr)
    y.free()
print(json.dumps(out))
