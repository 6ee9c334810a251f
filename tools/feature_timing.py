"""Device-resident timings of the frame-wise features (SURVEY 8f rank 2) on a cfg-2 shaped batch, next to the
oracle (CPU, one process) on a small sample.  CUDA events around `reps` calls after warm-up.  The pitch trackers
run with fmin C2, fmax C7 and their other defaults (frame_length 2048, hop 512); their oracle sample is one clip.
The rhythm features, beat_track and onset detection (dense output) take the device onset envelope of the batch (431 frames per 10 s
clip) and their defaults;
``rhythm_bounds`` holds the tempogram kernel's least time on the card (output bytes at 3.35 TB/s, two packed FP64
transforms per frame at 34 TFLOP/s), and ``card`` the GPU's name and power limit read in the same run.

    python tools/feature_timing.py [clips=1024] [reps=10] > gpurun_out/feature_timing.json
"""
import json
import os
import subprocess
import sys
import time
import warnings

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np

import bench
import librosa_b200 as lb
import onset_oracle as OD
import pitch_oracle as PO
import rhythm_oracle as RO
from oracle import ref_np as O

clips = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 10
w = dict(bench.WORKLOADS["cfg2"], clips=clips)
host = bench.make_batch(w, 0)
ctx = lb.default_context()
dev = ctx.to_device(host)
sr = 22050
T = 1 + host.shape[-1] // 512
frames = clips * T
mel_db = lb.power_to_db(lb.feature.melspectrogram(y=dev, sr=sr))
mel_pw = lb.feature.melspectrogram(y=dev, sr=sr)
dev128 = ctx.to_device(host[:128])
oenv = lb.onset.onset_strength(y=dev, sr=sr)
oenv_host = oenv.get().copy()
tg_dev = lb.feature.tempogram(onset_envelope=oenv)


C2, C7 = 65.40639132514966, 2093.004522404789
PEAK_KW = dict(pre_max=1, post_max=1, pre_avg=4, post_avg=5, delta=0.07, wait=1)   # onset_detect's at 22050 / 512


def free(x):
    for a in (x if isinstance(x, tuple) else (x,)):
        if isinstance(a, lb.DeviceArray):
            a.free()


FEATURES = {
    "spectral_centroid": (lambda: lb.feature.spectral_centroid(y=dev, sr=sr), lambda y: O.spectral_centroid(y=y, sr=sr)),
    "spectral_bandwidth": (lambda: lb.feature.spectral_bandwidth(y=dev, sr=sr), lambda y: O.spectral_bandwidth(y=y, sr=sr)),
    "spectral_rolloff": (lambda: lb.feature.spectral_rolloff(y=dev, sr=sr), lambda y: O.spectral_rolloff(y=y, sr=sr)),
    "spectral_flatness": (lambda: lb.feature.spectral_flatness(y=dev), lambda y: O.spectral_flatness(y=y)),
    "spectral_contrast": (lambda: lb.feature.spectral_contrast(y=dev, sr=sr), lambda y: O.spectral_contrast(y=y, sr=sr)),
    "rms(y)": (lambda: lb.feature.rms(y=dev), lambda y: O.rms(y=y)),
    "zero_crossing_rate": (lambda: lb.feature.zero_crossing_rate(dev), lambda y: O.zero_crossing_rate(y)),
    "chroma_stft(tuning=0)": (lambda: lb.feature.chroma_stft(y=dev, sr=sr, tuning=0.0), lambda y: O.chroma_stft(y=y, sr=sr, tuning=0.0)),
    "chroma_stft(estimated tuning)": (lambda: lb.feature.chroma_stft(y=dev, sr=sr), lambda y: O.chroma_stft(y=y, sr=sr)),
    "onset_strength": (lambda: lb.onset.onset_strength(y=dev, sr=sr), lambda y: O.onset_strength(y=y, sr=sr)),
    "effects.hpss (128 clips)": (lambda: lb.effects.hpss(dev128), None),
    "pcen(mel)": (lambda: lb.pcen(mel_pw, sr=sr), None),
    "amplitude_to_db(mel)": (lambda: lb.amplitude_to_db(mel_pw), None),
    "yin(C2-C7)": (lambda: lb.yin(dev, fmin=C2, fmax=C7, sr=sr), lambda y: PO.yin(y, fmin=C2, fmax=C7, sr=sr)),
    "pyin(C2-C7)": (lambda: lb.pyin(dev, fmin=C2, fmax=C7, sr=sr), lambda y: PO.pyin(y, fmin=C2, fmax=C7, sr=sr)),
    "tempogram(onset_envelope)": (lambda: lb.feature.tempogram(onset_envelope=oenv),
                                  lambda y: RO.tempogram(onset_envelope=oenv_host[:len(y)])),
    "fourier_tempogram(onset_envelope)": (lambda: lb.feature.fourier_tempogram(onset_envelope=oenv),
                                          lambda y: RO.fourier_tempogram(onset_envelope=oenv_host[:len(y)])),
    "tempo(onset_envelope)": (lambda: lb.feature.tempo(onset_envelope=oenv),
                              lambda y: RO.tempo(onset_envelope=oenv_host[:len(y)])),
    "tempo(tg, aggregate=None)": (lambda: lb.feature.tempo(tg=tg_dev, aggregate=None), None),
    "onset_strength(aggregate=np.median)": (lambda: lb.onset.onset_strength(y=dev, sr=sr, aggregate=np.median), None),
    "beat_track(onset_envelope)": (lambda: lb.beat.beat_track(onset_envelope=oenv, sparse=False), None),
    "beat_track(onset_envelope, bpm=120)": (lambda: lb.beat.beat_track(onset_envelope=oenv, bpm=120.0, sparse=False),
                                            None),
    "plp(onset_envelope)": (lambda: lb.beat.plp(onset_envelope=oenv), None),
    "onset_detect(onset_envelope)": (lambda: lb.onset.onset_detect(onset_envelope=oenv, sparse=False),
                                     lambda y: OD.onset_detect(onset_envelope=oenv_host[:len(y)], sparse=False)),
    "onset_detect(y)": (lambda: lb.onset.onset_detect(y=dev, sr=sr, sparse=False), None),
    "peak_pick(dp_value)": (lambda: lb.util.peak_pick(oenv, sparse=False, method="dp_value", **PEAK_KW),
                            lambda y: OD.peak_pick(oenv_host[:len(y)], sparse=False, method="dp_value", **PEAK_KW)),
}
CPU_SAMPLE = {"yin(C2-C7)": 1, "pyin(C2-C7)": 1}   # clips in the oracle sample (default 8)


def rhythm_bounds(rows, n_frames, win=384):
    """Least time of the tempogram kernel on an H100 SXM from the data sheet: float64 output bytes at 3.35 TB/s,
    and 2 packed real transforms of N = 2^ceil(log2(2 win - 1)) points per frame (5 (N/2) log2(N/2) flops each,
    plus the un-mix) at 34 TFLOP/s FP64."""
    N = 1 << int(np.ceil(np.log2(2 * win - 1)))
    M = N // 2
    flops = rows * n_frames * 2 * (5 * M * np.log2(M) + 10 * M)
    nbytes = rows * n_frames * win * 8
    return {"bytes": nbytes, "flop": flops, "bytes_ms": nbytes / 3.35e12 * 1e3, "flop_ms": flops / 34e12 * 1e3}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[lb.default_context().device] if q.returncode == 0 else "unknown"


out = {"clips": clips, "frames": frames, "reps": reps, "card": card(),
       "rhythm_bounds": rhythm_bounds(clips, oenv.shape[-1]), "features": {}}
with warnings.catch_warnings():
    warnings.simplefilter("ignore")
    for name, (gpu, cpu) in FEATURES.items():
        for _ in range(3):
            free(gpu())
        ctx.synchronize()
        e0, e1 = ctx.event(), ctx.event()
        l0 = ctx.launch_count
        e0.record()
        for _ in range(reps):
            free(gpu())
        e1.record()
        ctx.synchronize()
        ms = e0.elapsed_ms(e1) / reps
        nfr = 128 * T if "128 clips" in name else frames
        row = {"gpu_ms": round(ms, 3), "frames": nfr, "gpu_frames_per_s": round(nfr / ms * 1e3),
               "launches_per_call": (ctx.launch_count - l0) / reps}
        if cpu is not None:
            sample = host[:CPU_SAMPLE.get(name, 8)]
            cpu(sample[:1])
            t0 = time.perf_counter()
            cpu(sample)
            dt = time.perf_counter() - t0
            row["cpu_oracle_frames_per_s_1proc"] = round(sample.shape[0] * T / dt)
            row["cpu_oracle_s_per_clip"] = round(dt / sample.shape[0], 4)
        out["features"][name] = row
        print(name, row, file=sys.stderr)
print(json.dumps(out, indent=1))
