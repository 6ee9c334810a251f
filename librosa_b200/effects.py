"""``librosa.effects.hpss`` / ``harmonic`` / ``percussive`` with librosa's signatures (reference:
librosa/effects.py:58-131, :134-206, :209-281): stft -> decompose.hpss -> istft, every intermediate on the
device (one upload of the signal, one download per returned component)."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _native as nat
from . import _pipeline as pl
from .core.spectrum import istft, phase_vocoder, stft
from .decompose import _hpss_device
from .util.exceptions import ParameterError

__all__ = ["hpss", "harmonic", "percussive", "time_stretch", "pitch_shift"]


def _separate(y, want, *, kernel_size, power, mask, margin, n_fft, hop_length, win_length, window, center, pad_mode):
    # NB: like the reference (effects.py:87-94, :102-119) `window` is accepted but not forwarded to stft / istft.
    if mask:
        raise nat.UnsupportedOnGPU("effects.hpss(mask=True) inverts the masks themselves; not supported on the GPU")
    n, req = pl.precheck_signal(y)
    with pl.Scope(y) as sc:
        staged = pl.StagedInput(y)
        D = sc.own(stft(sc.own(staged.dev), n_fft=n_fft, hop_length=hop_length, win_length=win_length, center=center,
                        pad_mode=pad_mode))
        staged.scan_uncovered(n_fft, hop_length, win_length, center, D.shape[-1])
        harm, perc = _hpss_device(sc, D, kernel_size=kernel_size, power=power, mask=False, margin=margin)
        D.free()
        outs = []
        for name, comp in (("harm", harm), ("perc", perc)):
            if name in want:
                yd_out = istft(comp, n_fft=n_fft, hop_length=hop_length, win_length=win_length, center=center, length=n)
                outs.append(sc.result(yd_out, req, validate=True))
            comp.free()
        return outs


def hpss(y, *, kernel_size=31, power: float = 2.0, mask: bool = False, margin=1.0, n_fft: int = 2048,
         hop_length: Optional[int] = None, win_length: Optional[int] = None, window="hann", center: bool = True,
         pad_mode="constant"):
    """Decompose a signal into harmonic and percussive components; same contract as ``librosa.effects.hpss``."""
    h, p = _separate(y, ("harm", "perc"), kernel_size=kernel_size, power=power, mask=mask, margin=margin, n_fft=n_fft,
                     hop_length=hop_length, win_length=win_length, window=window, center=center, pad_mode=pad_mode)
    return h, p


def harmonic(y, *, kernel_size=31, power: float = 2.0, mask: bool = False, margin=1.0, n_fft: int = 2048,
             hop_length: Optional[int] = None, win_length: Optional[int] = None, window="hann", center: bool = True,
             pad_mode="constant"):
    """Harmonic component of a signal; same contract as ``librosa.effects.harmonic``."""
    return _separate(y, ("harm",), kernel_size=kernel_size, power=power, mask=mask, margin=margin, n_fft=n_fft,
                     hop_length=hop_length, win_length=win_length, window=window, center=center, pad_mode=pad_mode)[0]


def percussive(y, *, kernel_size=31, power: float = 2.0, mask: bool = False, margin=1.0, n_fft: int = 2048,
               hop_length: Optional[int] = None, win_length: Optional[int] = None, window="hann", center: bool = True,
               pad_mode="constant"):
    """Percussive component of a signal; same contract as ``librosa.effects.percussive``."""
    return _separate(y, ("perc",), kernel_size=kernel_size, power=power, mask=mask, margin=margin, n_fft=n_fft,
                     hop_length=hop_length, win_length=win_length, window=window, center=center, pad_mode=pad_mode)[0]


def time_stretch(y, *, rate: float, **kwargs):
    """Time-stretch a signal by ``rate`` (stft -> phase_vocoder -> istft, all on the device); same contract as
    ``librosa.effects.time_stretch`` (effects.py:284-361).  ``kwargs`` go to ``stft`` and ``istft``."""
    if rate <= 0:
        raise ParameterError("rate must be a positive number")
    n, req = pl.precheck_signal(y)
    with pl.Scope(y) as sc:
        staged = pl.StagedInput(y)
        D = sc.own(stft(sc.own(staged.dev), **kwargs))
        staged.scan_uncovered(kwargs.get("n_fft", 2048), kwargs.get("hop_length"), kwargs.get("win_length"),
                              kwargs.get("center", True), D.shape[-1])
        # the reference forwards these two (deprecated, unused) arguments, so its call always warns; same here
        Ds = sc.own(phase_vocoder(D, rate=rate, hop_length=kwargs.get("hop_length"), n_fft=kwargs.get("n_fft")))
        D.free()
        return sc.result(istft(Ds, length=round(n / rate), **kwargs), req, validate=True)


def pitch_shift(y, *, sr: float, n_steps: float, bins_per_octave: int = 12, res_type: str = "soxr_hq",
                scale: bool = False, **kwargs):
    """Shift the pitch of ``y`` by ``n_steps`` steps; same contract as ``librosa.effects.pitch_shift``
    (effects.py:487-574): time_stretch by ``2**(-n_steps / bins_per_octave)``, resample from ``sr / rate`` back to
    ``sr``, crop / zero-pad to the input length — all on the device.  Only ``res_type="polyphase"`` runs on the GPU
    (see ``resample``); like the reference it needs an integer ``sr / rate`` (whole octaves, ...) and raises
    ``ParameterError`` otherwise.  ``kwargs`` go to ``stft`` / ``istft``."""
    from .core.audio import resample
    from .util.utils import is_positive_int

    if not is_positive_int(bins_per_octave):
        raise ParameterError(f"bins_per_octave={bins_per_octave} must be a positive integer.")
    rate = 2.0 ** (-float(n_steps) / bins_per_octave)
    n, req = pl.precheck_signal(y)
    with pl.Scope(y) as sc:
        staged = pl.StagedInput(y)
        staged.scan_all()
        stretched = sc.own(time_stretch(sc.own(staged.dev), rate=rate, **kwargs))
        shifted = sc.own(resample(stretched, orig_sr=float(sr) / rate, target_sr=sr, res_type=res_type, scale=scale))
        stretched.free()
        # util.fix_length(y_shift, size=y.shape[-1]) on the device
        m = shifted.shape[-1]
        if m == n:
            out = shifted
        else:
            lead = shifted.shape[:-1]
            rows = pl.clip_count(lead)
            out = (sc.zeros if m < n else sc.empty)(tuple(lead) + (n,), np.float32)
            if rows and min(m, n):
                nat.check(nat.lib().b2l_copy2d(sc.ctx.handle, C.c_void_p(out.ptr), n * 4, C.c_void_p(shifted.ptr),
                                               m * 4, min(m, n) * 4, rows))
        return sc.result(out, req, validate=True)
