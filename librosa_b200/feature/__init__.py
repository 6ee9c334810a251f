"""``librosa.feature`` names of the FFT time-frequency path, of its frame-wise consumers, of the rhythm features and of
the feature-stacking utilities."""
from . import inverse
from .rhythm import fourier_tempogram, tempo, tempogram
from .spectral import chroma_cens, chroma_cqt, chroma_stft, chroma_vqt, melspectrogram, mfcc, tonnetz
from .stats import (rms, spectral_bandwidth, spectral_centroid, spectral_contrast, spectral_flatness,
                    spectral_rolloff, zero_crossing_rate)
from .utils import delta, stack_memory

__all__ = ["inverse", "melspectrogram", "mfcc", "chroma_stft", "chroma_cqt", "chroma_cens", "chroma_vqt", "tonnetz", "spectral_centroid", "spectral_bandwidth", "spectral_rolloff",
           "spectral_flatness", "spectral_contrast", "rms", "zero_crossing_rate",
           "tempogram", "fourier_tempogram", "tempo", "delta", "stack_memory"]
