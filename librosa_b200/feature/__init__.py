"""``librosa.feature`` names of the FFT time-frequency path, of its frame-wise consumers and of the rhythm features."""
from . import inverse
from .rhythm import fourier_tempogram, tempo, tempogram
from .spectral import chroma_stft, melspectrogram, mfcc
from .stats import (rms, spectral_bandwidth, spectral_centroid, spectral_contrast, spectral_flatness,
                    spectral_rolloff, zero_crossing_rate)

__all__ = ["inverse", "melspectrogram", "mfcc", "chroma_stft", "spectral_centroid", "spectral_bandwidth", "spectral_rolloff",
           "spectral_flatness", "spectral_contrast", "rms", "zero_crossing_rate",
           "tempogram", "fourier_tempogram", "tempo"]
