"""Device-resident timings of the frame-wise features (SURVEY 8f rank 2) on a cfg-2 shaped batch, next to the
oracle (CPU, one process) on a small sample.  CUDA events around `reps` calls after warm-up.  The pitch trackers
run with fmin C2, fmax C7 and their other defaults (frame_length 2048, hop 512); their oracle sample is one clip.
The rhythm features, beat_track and onset detection (dense output) take the device onset envelope of the batch (431 frames per 10 s
clip) and their defaults;
``rhythm_bounds`` holds the tempogram kernel's least time on the card (output bytes at 3.35 TB/s, two packed FP64
transforms per frame at 34 TFLOP/s), and ``card`` the GPU's name and power limit read in the same run.  ``sequence``
times the HMM decoders on their own device-resident float32 shapes (independent of ``clips``), each with its least
time from the shapes (predecessor visits x frames as FP64 add-compares at 34 TFLOP/s; bytes of prob, back-pointers
and states at 3.35 TB/s) and the oracle's CPU time per clip.  ``alignment`` times dtw (device float32 features,
cost matrix, accumulation and path) and rqa (device float32 similarity, score and path), each with its least time from
the shapes: about 20 bytes per cell (C, D, steps) for dtw and 1 + 2 * 4 per cell for rqa at 3.35 TB/s, and the
number of anti-diagonals the cells' dependency chain must pass through one after another.

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
import sequence_oracle as SQ
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


def sequence_timings():
    rng = np.random.default_rng(0)
    loop25, local720 = lb.sequence.transition_loop(25, 0.9), lb.sequence.transition_local(720, 31)
    dense = rng.random((1024, 1024))
    dense /= dense.sum(axis=1, keepdims=True)
    binary = np.array([[0.9, 0.1], [0.2, 0.8]])
    p25 = rng.random((1024, 25, 431)).astype(np.float32)
    p25 /= p25.sum(axis=-2, keepdims=True)
    # name: (prob shape, call on a device prob, problems, states per problem, predecessor visits per frame, oracle)
    cases = {
        "viterbi_discriminative(25 states, loop)": (p25, lambda x: lb.sequence.viterbi_discriminative(x, loop25),
                                                    1024, 25, 25 * 25, "disc", loop25, {}),
        "viterbi(1024 states, dense)": ((64, 1024, 1000), lambda x: lb.sequence.viterbi(x, dense), 64, 1024,
                                        1024 * 1024, "viterbi", dense, {}),
        "viterbi(transition_local(720, 31), min_prob=1e-4)": (
            (1024, 720, 431), lambda x: lb.sequence.viterbi(x, local720, transition_min_prob=1e-4), 1024, 720,
            int((np.log(local720 + np.finfo(np.float32).tiny) >= np.log(1e-4 + np.finfo(np.float32).tiny)).sum()),
            "viterbi", local720, dict(transition_min_prob=1e-4)),
        "viterbi_binary(88 labels)": ((1024, 88, 431), lambda x: lb.sequence.viterbi_binary(x, binary), 1024 * 88, 2,
                                      4, "binary", binary, {}),
    }
    res = {}
    for name, (shape, call, problems, S, visits, op, trans, kw) in cases.items():
        host_p = shape if isinstance(shape, np.ndarray) else rng.random(shape).astype(np.float32)
        x = ctx.to_device(host_p)
        call(x)
        ctx.synchronize()
        e0, e1 = ctx.event(), ctx.event()
        l0 = ctx.launch_count
        e0.record()
        n = max(1, reps // 5) if S >= 720 else reps
        for _ in range(n):
            call(x)
        e1.record()
        ctx.synchronize()
        ms = e0.elapsed_ms(e1) / n
        T_ = host_p.shape[-1]
        ops = 2.0 * visits * T_ * (problems // (88 if op == "binary" else 1)) * (88 if op == "binary" else 1)
        nbytes = host_p.nbytes + problems * (2 * S * T_ + 2 * T_)
        t0 = time.perf_counter()
        SQ.run(op, host_p[0], trans, **kw)
        cpu = time.perf_counter() - t0
        res[name] = {"gpu_ms": round(ms, 3), "launches_per_call": (ctx.launch_count - l0) / n,
                     "least_ms_fp64": round(ops / 34e12 * 1e3, 3), "least_ms_bytes": round(nbytes / 3.35e12 * 1e3, 3),
                     "cpu_oracle_s_per_clip": round(cpu, 4)}
        print(name, res[name], file=sys.stderr)
        x.free()
    return res


def alignment_timings():
    rng = np.random.default_rng(0)
    cases = {}
    for N, M in ((4000, 4500), (20000, 20000)):
        X = ctx.to_device(rng.random((12, N)).astype(np.float32))
        Y = ctx.to_device(rng.random((12, M)).astype(np.float32))
        cases[f"dtw(12 x {N}, 12 x {M})"] = (lambda X=X, Y=Y: lb.sequence.dtw(X, Y), N, M, 20, (X, Y))
    sim = ctx.to_device((rng.random((4000, 4000)) > 0.7).astype(np.float32))
    cases["rqa(4000 x 4000, float32)"] = (lambda: lb.sequence.rqa(sim), 4000, 4000, 9, (sim,))
    res = {}
    for name, (call, N, M, per_cell, keep) in cases.items():
        free(call())
        ctx.synchronize()
        n = 3 if N * M > 1e8 else 10
        e0, e1 = ctx.event(), ctx.event()
        l0 = ctx.launch_count
        e0.record()
        for _ in range(n):
            free(call())
        e1.record()
        ctx.synchronize()
        ms = e0.elapsed_ms(e1) / n
        res[name] = {"gpu_ms": round(ms, 3), "launches_per_call": (ctx.launch_count - l0) / n,
                     "gcells_per_s": round(N * M / ms / 1e6, 2),
                     "least_ms_bytes": round(N * M * per_cell / 3.35e12 * 1e3, 3), "anti_diagonals": N + M - 1}
        print(name, res[name], file=sys.stderr)
        for a in keep:
            a.free()
    return res


out["sequence"] = sequence_timings()
out["alignment"] = alignment_timings()
print(json.dumps(out, indent=1))
