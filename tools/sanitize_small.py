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
# fused mel front end: one hop per instance window of the power-of-two kernel (sr 22 050, 128 mels), n_fft 64 (the
# slack after the last power row), the mixed-radix kernel with 16 and 32 lanes per frame, mfcc with KS = 1 and 2
for n_fft, hop in [(1024, 608), (1024, 626), (2048, 1001), (2048, 1111), (2048, 1112), (4096, 618), (4096, 1120),
                   (4096, 1121), (8192, 2048), (64, 16), (400, 160), (2400, 600)]:
    yb = (0.1 * rng.standard_normal((3, 8 * hop + n_fft))).astype(np.float32)
    M = lb.feature.melspectrogram(y=yb, sr=22050, n_fft=n_fft, hop_length=hop)
    print(n_fft, hop, M.shape, bool(np.isfinite(M).all()))
for n_mels, n_mfcc in [(128, 20), (13, 20)]:
    C = lb.feature.mfcc(y=y, sr=22050, n_fft=512, hop_length=128, n_mels=n_mels, n_mfcc=n_mfcc)
    print("mfcc", n_mels, n_mfcc, C.shape, bool(np.isfinite(C).all()))
# b2l_mfcc with a caller's scratch one float off 16-byte alignment: dct_clamp4_kernel streams its tiles in 4-byte pieces
import ctypes
from librosa_b200 import _native as nat, _pipeline as pl
from librosa_b200.feature import spectral as S
ctx = lb.default_context()
w, wkey = pl.resolve_window("hann", 512, 512)
basis, bkey = pl.mel_basis(22050, 512, {})
dct = S._dct_basis(128, 20, 2, "ortho", 0)
plan = nat.make_plan(ctx, ("mfcc", 512, 128, True, "constant", wkey, bkey, 2.0, pl.digest(dct)), n_fft=512,
                     hop_length=128, center=True, pad_mode="constant", window=w, mel_basis=basis, power=2.0,
                     dct_basis=dct, amin=1e-10, ref_value=1.0, top_db=80.0)
T = plan.n_frames(y.shape[-1])
d_y = lb.to_device(y)
out = lb.DeviceArray.empty(ctx, (y.shape[0] * 20 * T + 1,), np.float32)
scr = lb.DeviceArray.empty(ctx, (y.shape[0] * 128 * ((T + 63) // 64 * 64) + 1,), np.float32)
nat.check(nat.lib().b2l_mfcc(ctx.handle, plan.handle, ctypes.c_void_p(d_y.ptr), y.shape[0], y.shape[-1], y.shape[-1],
                             ctypes.c_void_p(out.ptr + 4), ctypes.c_void_p(scr.ptr + 4)))
Cu = out.get()[1:].reshape(y.shape[0], 20, T)
print("mfcc unaligned scratch", Cu.shape, bool(np.array_equal(Cu, lb.feature.mfcc(y=y, sr=22050, n_fft=512, hop_length=128))))
# stft / spectrogram / fused statistics: one hop per instance window of MODE_STFT / MODE_SPEC and of MODE_STATS (the
# last hop of each), and stats_kernel at the top of its warp ladder (29 056 bins, one warp per block)
from librosa_b200.core.spectrum import _spectrogram
for n_fft, hop in [(1024, 674), (1024, 686), (2048, 1248), (2048, 1303), (2048, 5206), (4096, 1546), (4096, 1915),
                   (4096, 10101), (8192, 16672)]:
    yb = (0.1 * rng.standard_normal((2, 4 * hop + n_fft))).astype(np.float32)
    D = lb.stft(yb, n_fft=n_fft, hop_length=hop)
    Sp, _ = _spectrogram(y=yb, n_fft=n_fft, hop_length=hop, power=1.5)
    print("stft", n_fft, hop, D.shape, bool(np.isfinite(D).all() and np.isfinite(Sp).all()))
for n_fft, hop in [(1024, 652), (1024, 665), (2048, 1165), (2048, 1230), (2048, 5051), (4096, 1194), (4096, 1613),
                   (4096, 9408), (8192, 12544)]:
    yb = (0.1 * rng.standard_normal((2, 4 * hop + n_fft))).astype(np.float32)
    c = lb.feature.spectral_centroid(y=yb, sr=22050, n_fft=n_fft, hop_length=hop)
    print("stats", n_fft, hop, c.shape, bool(np.isfinite(c).all()))
Sb = np.abs(rng.standard_normal((2, 29056, 3))).astype(np.float32)
print("stats_kernel 29056 bins", bool(np.isfinite(lb.feature.spectral_centroid(S=Sb, sr=22050)).all()))
print("sanitize_small done")
