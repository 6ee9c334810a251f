"""``librosa.util`` names used on the FFT time-frequency path, ``peak_pick``, ``fill_off_diagonal`` and the peak test
``localmax`` / ``localmin``."""
from .exceptions import LibrosaError, ParameterError
from .peak import peak_pick
from .utils import (
    MAX_MEM_BLOCK,
    abs2,
    dtype_c2r,
    dtype_r2c,
    expand_to,
    fill_off_diagonal,
    fix_length,
    frame,
    is_positive_int,
    localmax,
    localmin,
    normalize,
    pad_center,
    tiny,
    valid_audio,
)

__all__ = [
    "LibrosaError", "ParameterError", "MAX_MEM_BLOCK", "abs2", "dtype_c2r", "dtype_r2c", "expand_to",
    "fill_off_diagonal", "fix_length", "frame", "is_positive_int", "localmax", "localmin", "normalize", "pad_center", "peak_pick", "tiny", "valid_audio",
]
