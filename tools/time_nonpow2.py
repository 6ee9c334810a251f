"""Device-resident timing of frame lengths that are not a power of two: n_fft=400 / hop=160 / 80 mels, 1024 x 10 s
@ 16 kHz (the speech front-end shape), on the mixed-radix kernel (default) and on the chirp-z kernels (B2L_MR=0),
with the power-of-two 512 configuration beside them.  One JSON line per measurement."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, librosa_b200 as lb
ctx = lb.default_context()
y = (0.1 * np.random.default_rng(0).standard_normal((1024, 160000))).astype(np.float32)
yd = ctx.to_device(y)
cases = [("mel 400/160/80", lambda: lb.feature.melspectrogram(y=yd, sr=16000, n_fft=400, hop_length=160, n_mels=80)),
         ("mfcc 400/160/80->13", lambda: lb.feature.mfcc(y=yd, sr=16000, n_mfcc=13, n_fft=400, hop_length=160, n_mels=80)),
         ("stft 400/160", lambda: lb.stft(yd, n_fft=400, hop_length=160)),
         ("spectral_centroid 400/160", lambda: lb.feature.spectral_centroid(y=yd, sr=16000, n_fft=400, hop_length=160)),
         ("mel 800/160/80", lambda: lb.feature.melspectrogram(y=yd, sr=16000, n_fft=800, hop_length=160, n_mels=80)),
         ("mel 512/160/80", lambda: lb.feature.melspectrogram(y=yd, sr=16000, n_fft=512, hop_length=160, n_mels=80))]
Dd = lb.stft(yd, n_fft=400, hop_length=160)
cases.insert(3, ("istft 400/160", lambda: lb.istft(Dd, hop_length=160, n_fft=400, length=160000)))
for mr in ("1", "0"):
    if mr == "0" and os.environ.get("B2L_SKIP_CZT"):
        continue
    os.environ["B2L_MR"] = mr
    for name, fn in cases:
        if mr == "0" and "512" in name:
            continue
        for _ in range(3): fn().free()
        ctx.synchronize()
        e0, e1 = ctx.event(), ctx.event()
        e0.record()
        for _ in range(10): fn().free()
        e1.record(); ctx.synchronize()
        print(json.dumps({"what": name, "B2L_MR": mr, "ms": round(e0.elapsed_ms(e1) / 10, 3), "frames": 1024 * 1001}), flush=True)
