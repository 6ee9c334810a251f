"""``librosa.core`` names of the FFT time-frequency path."""
from .audio import resample, stream
from .convert import (fft_frequencies, fourier_tempo_frequencies, frames_to_samples, frames_to_time, hz_to_mel,
                      hz_to_octs, mel_frequencies, mel_to_hz, samples_to_time, tempo_frequencies)
from .pitch import estimate_tuning, pyin, yin
from .spectrum import (_spectrogram, amplitude_to_db, db_to_amplitude, db_to_power, griffinlim, istft, pcen,
                       phase_vocoder, power_to_db, reassigned_spectrogram, stft)

__all__ = ["stream", "resample", "stft", "istft", "griffinlim", "_spectrogram", "power_to_db", "amplitude_to_db", "pcen", "phase_vocoder", "reassigned_spectrogram", "db_to_power", "db_to_amplitude", "hz_to_mel", "mel_to_hz", "mel_frequencies",
           "fft_frequencies", "tempo_frequencies", "fourier_tempo_frequencies", "frames_to_samples", "frames_to_time", "samples_to_time", "hz_to_octs", "estimate_tuning", "yin", "pyin"]
