"""librosa_b200 — H100 (sm_90a) implementation of librosa's FFT time-frequency hot path.

Drop-in for this path only: ``import librosa_b200 as librosa`` gives ``stft``, ``istft``,
``power_to_db``, ``feature.melspectrogram``, ``feature.mfcc``, ``filters.mel / get_window /
window_sumsquare``, ``util.frame`` (and the small helpers around them) with librosa's signatures,
shapes, dtypes, warnings and exceptions.  The arithmetic runs in hand-written CUDA kernels reached
through a C ABI (``include/b2l.h``) with ctypes — no PyTorch, no Triton, no CPU fallback.
"""
from . import beat, core, decompose, effects, feature, filters, onset, util
from ._native import (
    Context,
    DeviceArray,
    NativeLibraryError,
    UnsupportedOnGPU,
    bind_host_to_device,
    default_context,
    device_count,
    pinned_empty,
)
from .core.audio import resample, stream
from .core.convert import (fft_frequencies, fourier_tempo_frequencies, frames_to_samples, frames_to_time, hz_to_mel,
                           hz_to_octs, mel_frequencies, mel_to_hz, samples_to_time, tempo_frequencies)
from .core.pitch import estimate_tuning, pyin, yin
from .core.spectrum import (_spectrogram, amplitude_to_db, db_to_amplitude, db_to_power, griffinlim, istft,
                            pcen, phase_vocoder, power_to_db, reassigned_spectrogram, stft)
from .util.exceptions import LibrosaError, ParameterError

__version__ = "0.1.0"


def device_copy(ctx, dst, dst_byte_offset, src):
    """Stream-ordered device-to-device copy of the DeviceArray ``src`` into ``dst`` at a byte offset (building a
    batch on the root GPU before a scatter)."""
    import ctypes as _C

    from . import _native as _nat

    if dst_byte_offset < 0 or dst_byte_offset + src.nbytes > dst.nbytes:
        raise ValueError("copy does not fit the destination")
    _nat.check(_nat.lib().b2l_d2d(ctx.handle, _C.c_void_p(dst.ptr + int(dst_byte_offset)), _C.c_void_p(src.ptr), src.nbytes))


def to_device(arr, device=None):
    """Copy a NumPy array to the GPU; device-resident inputs make every function return DeviceArrays."""
    return default_context(device).to_device(arr)


__all__ = [
    "stream", "resample", "stft", "istft", "griffinlim", "power_to_db", "amplitude_to_db", "pcen", "phase_vocoder", "reassigned_spectrogram", "db_to_power", "db_to_amplitude", "_spectrogram", "feature", "filters", "util", "core", "onset", "beat", "decompose", "effects",
    "hz_to_mel", "mel_to_hz", "hz_to_octs", "estimate_tuning", "yin", "pyin", "mel_frequencies", "fft_frequencies", "tempo_frequencies", "fourier_tempo_frequencies", "frames_to_samples", "frames_to_time", "samples_to_time", "ParameterError", "LibrosaError",
    "Context", "DeviceArray", "default_context", "device_count", "pinned_empty", "to_device", "device_copy",
    "NativeLibraryError", "UnsupportedOnGPU", "bind_host_to_device",
]
