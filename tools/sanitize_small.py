"""Small forward / inverse calls for compute-sanitizer (memcheck / racecheck) runs."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import librosa_b200 as lb

rng = np.random.default_rng(0)
y = (0.1 * rng.standard_normal((3, 9000))).astype(np.float32)
for n_fft, hop in [(2048, 512), (1024, 256), (4096, 1024), (512, 128), (256, 64)]:
    D = lb.stft(y, n_fft=n_fft, hop_length=hop)
    M = lb.feature.melspectrogram(y=y, sr=22050, n_fft=n_fft, hop_length=hop, n_mels=64)
    C = lb.feature.mfcc(y=y, sr=22050, n_fft=n_fft, hop_length=hop, n_mfcc=13, n_mels=64)
    c = lb.feature.spectral_centroid(y=y, sr=22050, n_fft=n_fft, hop_length=hop)
    yr = lb.istft(D, hop_length=hop, length=y.shape[-1])
    print(n_fft, D.shape, M.shape, C.shape, c.shape, float(np.abs(yr - y).max()))
# inverse geometries: a batch cut into several slots (halo rebuild), an odd hop (scalar gather loop), hop > n_fft (no carry)
for n_fft, hop, clips in [(2048, 512, 64), (512, 171, 3), (256, 300, 3)]:
    yb = np.tile(y, (clips // 3 + 1, 1))[:clips]
    yr = lb.istft(lb.stft(yb, n_fft=n_fft, hop_length=hop), hop_length=hop, length=yb.shape[-1])
    print(n_fft, hop, yr.shape, bool(np.isfinite(yr).all()))
print("sanitize_small done")
