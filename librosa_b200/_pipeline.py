"""Shared host logic between the public functions and the C ABI: argument normalisation, plan keys,
device staging of inputs / outputs.  Everything numeric happens in libb2l.so."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import warnings
from functools import lru_cache
from typing import NamedTuple, Tuple

import numpy as np

from . import _native as nat
from . import filters
from .util.exceptions import ParameterError
from .util.utils import is_positive_int, pad_center

_UNSUPPORTED_PAD = ("wrap", "maximum", "mean", "median", "minimum")   # librosa/core/spectrum.py:253


def float64_policy() -> str:
    """``B2L_FLOAT64``: what happens to float64 / complex128 data.

    * "native" (default) — the hot-path functions (stft, istft, _spectrogram, melspectrogram, mfcc,
      power_to_db) compute in FP64 on the GPU like the reference does (``_f64.py``); the wider functions,
      which have float32 kernels only, fall back to "downcast" for such inputs;
    * "downcast" — compute in float32, return arrays of the dtype librosa would return, warn once;
    * "quiet" — "downcast" without the warning;
    * "error" — refuse (``UnsupportedOnGPU``)."""
    return os.environ.get("B2L_FLOAT64", "native").lower()


def native_float64(dtype) -> bool:
    """True when data of this dtype should take the FP64 kernels."""
    return np.dtype(dtype) in (np.dtype(np.float64), np.dtype(np.complex128)) and float64_policy() == "native"


_warned_float64 = False


def _note_float64(what: str, stacklevel: int = 4):
    global _warned_float64
    if float64_policy() in ("downcast", "native") and not _warned_float64:
        _warned_float64 = True
        warnings.warn(f"{what}: float64 data is computed in float32 by this function on the GPU (results agree with "
                      "librosa to about 1e-6 relative, not to float64 precision; stft / istft / melspectrogram / mfcc "
                      "/ power_to_db have FP64 kernels); set B2L_FLOAT64=error to refuse instead, or B2L_FLOAT64=quiet "
                      "to silence this warning", stacklevel=stacklevel)


def check_real_dtype(dtype, what: str, native_ok: bool = False, stacklevel: int = 4) -> np.dtype:
    """``native_ok``: the caller has an FP64 path for float64 data (no downcast, no warning); ``stacklevel``: of
    the downcast warning, counted from ``_note_float64``."""
    dtype = np.dtype(dtype)
    if dtype == np.float32:
        return dtype
    if np.issubdtype(dtype, np.floating):
        if native_ok and dtype == np.float64 and float64_policy() == "native":
            return dtype
        if float64_policy() == "error":
            raise nat.UnsupportedOnGPU(
                f"{what}: dtype {dtype} is not supported by the float32 sm_90a kernels and B2L_FLOAT64=error "
                "(there is no CPU fallback)")
        _note_float64(what, stacklevel)
        return dtype
    raise ParameterError(f"{what}: data must be floating-point, got {dtype}")


def wide_complex_ok(what: str) -> bool:
    """complex128 requests served by the float32 kernels (stft dtype= on float32 data) under the float64 policy."""
    if float64_policy() == "error":
        return False
    _note_float64(what)
    return True


def digest(arr: np.ndarray) -> str:
    return hashlib.blake2b(np.ascontiguousarray(arr).tobytes(), digest_size=16).hexdigest()


def resolve_window(window, win_length: int, n_fft: int) -> Tuple[np.ndarray, str]:
    """get_window + pad_center exactly as librosa.stft does (core/spectrum.py:243-246)."""
    w = filters.get_window(window, win_length, fftbins=True)
    w = pad_center(np.asarray(w, dtype=np.float64), size=n_fft)
    return w, digest(w)


@lru_cache(maxsize=64)
def _mel_cached(sr, n_fft, items):
    kwargs = dict(items)
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        basis = filters.mel(sr=sr, n_fft=n_fft, **kwargs)
    basis.setflags(write=False)
    return basis, digest(basis), tuple(str(w.message) for w in caught)


def mel_basis(sr, n_fft, kwargs) -> Tuple[np.ndarray, str]:
    """filters.mel with memoisation (the reference recomputes it on every call, feature/spectral.py:2158)."""
    items = []
    for k, v in sorted(kwargs.items()):
        if k == "dtype":
            v = np.dtype(v).str
        items.append((k, v))
    try:
        basis, dg, msgs = _mel_cached(float(sr), int(n_fft), tuple(items))
    except TypeError:  # unhashable kwarg -> no memoisation
        basis = filters.mel(sr=sr, n_fft=n_fft, **kwargs)
        return basis, digest(basis)
    for m in msgs:
        warnings.warn(m, stacklevel=3)
    return basis, dg


def frame_params(n_fft, hop_length, win_length):
    """Defaults and the hop check of librosa/core/spectrum.py:231-237."""
    if win_length is None:
        win_length = n_fft
    if hop_length is None:
        hop_length = int(win_length // 4)
    elif not is_positive_int(hop_length):
        raise ParameterError(f"hop_length={hop_length} must be a positive integer")
    return int(hop_length), int(win_length)


def check_stft_geometry(n: int, n_fft: int, center: bool, pad_mode):
    """Padding-mode and length checks of librosa/core/spectrum.py:252-271, 329-333."""
    if center:
        if callable(pad_mode):
            raise nat.UnsupportedOnGPU("callable pad_mode cannot run on the GPU (no CPU fallback)")
        if pad_mode in _UNSUPPORTED_PAD:
            raise ParameterError(f"pad_mode='{pad_mode}' is not supported by librosa.stft")
        if pad_mode not in nat.PAD_MODES:
            raise ValueError(f"mode '{pad_mode}' is not supported")   # what np.pad raises
        if n_fft > n:
            warnings.warn(f"n_fft={n_fft} is too large for input signal of length={n}", stacklevel=5)
    elif n_fft > n:
        raise ParameterError(
            f"n_fft={n_fft} is too large for uncentered analysis of input signal of length={n}")
    return pad_mode if (center and isinstance(pad_mode, str)) else "constant"


def precheck_signal(y, native_ok: bool = False, stacklevel: int = 4):
    """Host-side validation of an input signal, done before any GPU resource is touched so that
    argument errors surface exactly as in the reference (util.valid_audio, core/spectrum.py:240).
    Returns ``(length, requested dtype)``.  ``native_ok``: the caller has an FP64 path."""
    if isinstance(y, nat.DeviceArray):
        if native_ok and y.dtype == np.float64 and y.layout == "c" and y.ndim > 0:
            return y.shape[-1], np.dtype(np.float64)
        if y.dtype != np.float32 or y.layout != "c":
            raise ParameterError("device input must be a C-ordered float32 DeviceArray")
        if y.ndim == 0:
            raise ParameterError("Audio data must be at least one-dimensional")
        return y.shape[-1], np.dtype(np.float32)
    # util.valid_audio's type / dtype / ndim checks on the host; its O(n) np.isfinite(y).all() pass runs on
    # the GPU instead (status word set by the kernels, see StagedInput).
    if not isinstance(y, np.ndarray):
        raise ParameterError("Audio data must be of type numpy.ndarray")
    if not np.issubdtype(y.dtype, np.floating):
        raise ParameterError("Audio data must be floating-point")
    if y.ndim == 0:
        raise ParameterError(f"Audio data must be at least one-dimensional, given y.shape={y.shape}")
    return y.shape[-1], check_real_dtype(y.dtype, "input signal", native_ok, stacklevel)


MIN_N_FFT, MAX_N_FFT = 8, 8192   # powers of two: kMinLog2M / kMaxLog2M in csrc/internal.h
MAX_CZT_N_FFT = 2047               # other sizes: Bluestein with P = 2^ceil(log2(2 n_fft - 1)) <= 4096
MAX_MR_N_FFT = 4096                # even sizes with a 5-smooth half: mixed-radix kernels (forward and inverse)


def is_pow2(n: int) -> bool:
    return n > 0 and (n & (n - 1)) == 0


def mr_covers(n_fft: int) -> bool:
    """True when the mixed-radix kernel (csrc/mr_kernel.cuh) takes the forward transform: even n_fft that is not a
    power of two and whose half has no prime factor above 5 (400, 320, 480, 800, 960, 1200, ...).  Mirror of
    ``mr_factor`` in csrc/plan.cu; ``B2L_MR=0`` sends these sizes back to the chirp-z kernels."""
    n_fft = int(n_fft)
    if is_pow2(n_fft) or n_fft < 12 or n_fft > MAX_MR_N_FFT or (n_fft & 1):
        return False
    if os.environ.get("B2L_MR", "") not in ("", "1"):
        return False
    m = n_fft // 2
    for q in (5, 3, 2):
        while m % q == 0:
            m //= q
    return m == 1


def fused_front_end(n_fft: int) -> bool:
    """Frame lengths whose melspectrogram / mfcc run as ONE fused kernel (+ the DCT kernel): powers of two
    (fwd_kernel) and the mixed-radix sizes (mr_kernel).  Everything else composes the spectrogram kernel with the
    ``S=`` kernels on the device."""
    return is_pow2(n_fft) or mr_covers(n_fft)


def require_supported_n_fft(n_fft: int, inverse: bool = False):
    """Power-of-two n_fft in [8, 8192] runs on the packed real-FFT kernels; even n_fft up to 4096 whose half is
    5-smooth (400, 480, 960, 1200, 3000, ...) on the mixed-radix kernels; any other n_fft in [3, 2047] (the
    reference tests' 501 / 1023 / 1025, ...) on the chirp-z kernels (forward and inverse).  Everything else
    librosa accepts is refused loudly by the float32 path — there is no CPU fallback (host float32 data of such
    sizes takes the FP64 kernels, see ``wide_route``)."""
    n_fft = int(n_fft)
    if is_pow2(n_fft):
        if MIN_N_FFT <= n_fft <= MAX_N_FFT:
            return
        raise nat.UnsupportedOnGPU(
            f"n_fft={n_fft}: the sm_90a kernels are built for powers of two from {MIN_N_FFT} to {MAX_N_FFT} "
            "(no CPU fallback)")
    if not (3 <= n_fft <= MAX_CZT_N_FFT) and not mr_covers(n_fft):
        raise nat.UnsupportedOnGPU(f"n_fft={n_fft}: non-power-of-two sizes are supported from 3 to {MAX_CZT_N_FFT}, and "
                                   f"even sizes up to {MAX_MR_N_FFT} whose half has no prime factor above 5 "
                                   "(no CPU fallback)")


def f32_kernels_cover(n_fft: int) -> bool:
    """True when the float32 hot-path kernels are built for this frame length."""
    n_fft = int(n_fft)
    if is_pow2(n_fft):
        return MIN_N_FFT <= n_fft <= MAX_N_FFT
    return 3 <= n_fft <= MAX_CZT_N_FFT or mr_covers(n_fft)


def wide_route(y, req_dtype, n_fft: int) -> bool:
    """Should this call take the FP64 kernels?  Yes for float64 data under the "native" policy, and for float32
    HOST data whose n_fft the float32 kernels are not built for (2^14 ... 2^20, non-powers of two above 2047):
    librosa accepts any frame length (its tests go to 2^16, tests/test_core.py:308-314), so those sizes run on
    the FP64 kernels and the result is rounded to the dtype librosa would return."""
    from . import _f64

    if np.dtype(req_dtype) == np.float64 and native_float64(req_dtype):
        return True
    return (not isinstance(y, nat.DeviceArray)) and not f32_kernels_cover(n_fft) and _f64.supported(n_fft)


def context_for(x):
    return x.ctx if isinstance(x, nat.DeviceArray) else nat.default_context()


def f64_constant(ctx, key, arr) -> int:
    """Device copy of a float64 / integer table cached by the context (Context.constant stores raw 4-byte words)."""
    arr = np.ascontiguousarray(arr)
    return ctx.constant(key, lambda: arr.reshape(-1).view(np.float32))


def clip_count(lead) -> int:
    """Number of clips in a batch with leading dimensions ``lead`` (one for a single clip)."""
    return int(np.prod(lead, dtype=np.int64)) if lead else 1


def frame_count(n: int, n_fft: int, hop: int, center: bool) -> int:
    """STFT frames of an ``n``-sample signal (Appendix A.1; librosa pads ``n_fft // 2`` on each side when centred)."""
    return 1 + (n + (2 * (n_fft // 2) if center else 0) - n_fft) // hop


class Front(NamedTuple):
    n: int
    dtype: np.dtype
    hop: int
    window: np.ndarray
    wkey: str
    mode: str
    n_frames: int


def forward_front(y, n_fft, hop_length, win_length, window, center, pad_mode, native_ok=True) -> Front:
    """Argument checks of a forward op (stft, _spectrogram, melspectrogram, mfcc, the spectral statistics) in the
    reference's order — hop, util.valid_audio, window, padding — before any GPU resource is touched."""
    hop, win_length = frame_params(n_fft, hop_length, win_length)
    n, dtype = precheck_signal(y, native_ok, stacklevel=5)
    win, wkey = resolve_window(window, win_length, n_fft)
    mode = check_stft_geometry(n, n_fft, center, pad_mode)
    return Front(n, dtype, hop, win, wkey, mode, frame_count(n, n_fft, hop, center))


# --------------------------------------------------------------------------------------------- status word
def status_word(ctx) -> int:
    """The context's status word once its stream has drained: bit 0 — a kernel saw a non-finite input sample
    (the device half of util.valid_audio), bit 1 — a negative spectrogram entry."""
    flag = C.c_int(0)
    nat.check(nat.lib().b2l_status_read(ctx.handle, C.byref(flag)))
    return flag.value


_NOT_FINITE = "Audio buffer is not finite everywhere"


def finish(dev: nat.DeviceArray, dtype=None, validate: bool = False) -> np.ndarray:
    """Copy a device result to a NumPy array of its logical shape (a swapped view for "ft"), free it and cast it
    to ``dtype``; ``validate``: raise like util.valid_audio when a kernel flagged a non-finite sample."""
    arr = dev.get()
    dev.free()
    if validate and status_word(dev.ctx) & 1:
        raise ParameterError(_NOT_FINITE)
    if dtype is not None and arr.dtype != dtype:
        arr = arr.astype(dtype)
    return arr


def _uncovered_begin(n_fft: int, hop: int, center: bool, n_frames: int) -> int:
    """First sample that no frame reads; 0 when hop > n_fft leaves gaps between the frames."""
    return 0 if hop > n_fft else max(0, (n_frames - 1) * hop + n_fft - (n_fft // 2 if center else 0))


class StagedInput:
    """A signal batch resident on the device as ``[n_clips][n]`` (call precheck_signal first).

    For a host signal this object also runs util.valid_audio's finite check on the device: the upload resets the
    context's status word, the kernels flag the samples they read, ``scan_uncovered`` / ``scan_all`` cover the
    rest, and ``result`` reads the verdict with the result.  Device signals are returned as they are computed."""

    def __init__(self, y, dtype=np.float32):
        self.ctx = context_for(y)
        self.on_device = isinstance(y, nat.DeviceArray)
        if self.on_device:
            self.dev = y
        else:
            nat.check(nat.lib().b2l_status_reset(self.ctx.handle))
            host = np.ascontiguousarray(y, dtype=dtype)
            self.dev = nat.DeviceArray.empty(self.ctx, host.shape, dtype)
            if host.nbytes:
                nat.check(nat.lib().b2l_h2d(self.ctx.handle, C.c_void_p(self.dev.ptr),
                                            host.ctypes.data_as(C.c_void_p), host.nbytes))
            self._host = host   # keep alive until the stream has consumed it
        self.lead = self.dev.shape[:-1]
        self.n = self.dev.shape[-1]
        self.n_clips = clip_count(self.lead)

    def _scan(self, begin: int):
        if not self.on_device and self.n_clips and begin < self.n:
            nat.check(nat.lib().b2l_scan_finite(self.ctx.handle, C.c_void_p(self.dev.ptr), self.n_clips, self.n,
                                                self.n, begin))

    def scan_uncovered(self, n_fft: int, hop_length, win_length, center: bool, n_frames: int):
        """Scan the samples that no STFT frame reads (the tail after the last frame, or everything when the hop
        leaves gaps); ``hop_length`` / ``win_length`` as passed to stft (None: the defaults)."""
        hop, _ = frame_params(n_fft, hop_length, win_length)
        self._scan(_uncovered_begin(n_fft, hop, center, n_frames))

    def scan_all(self):
        """Scan every sample (for consumers that do not flag what they read)."""
        self._scan(0)

    def release(self):
        """Free the upload of a host signal right after the work on it is enqueued (a device signal stays)."""
        if not self.on_device:
            self.dev.free()

    def check_finite(self):
        if not self.on_device and status_word(self.ctx) & 1:
            raise ParameterError(_NOT_FINITE)

    def result(self, dev: nat.DeviceArray, dtype=None):
        """The caller's return value: ``dev`` itself for a device signal, else a NumPy array of ``dtype``,
        validated with the status verdict."""
        return dev if self.on_device else finish(dev, dtype, validate=True)


# --------------------------------------------------------------------------------------------- spectrogram inputs
def spectrogram_input(S):
    """A real spectrogram-like argument ``(..., rows, frames)``, host or device -> (DeviceArray, requested dtype,
    input was on the device).  Host arrays are uploaded C-ordered; device arrays keep their layout."""
    if isinstance(S, nat.DeviceArray):
        if S.dtype != np.float32:
            raise ParameterError("device spectrogram must be float32")
        return S, np.dtype(np.float32), True
    S = np.asarray(S)
    if np.iscomplexobj(S):
        raise ParameterError("spectrogram input must be real")
    req = check_real_dtype(S.dtype if np.issubdtype(S.dtype, np.floating) else np.float32, "S")
    return nat.default_context().to_device(np.ascontiguousarray(S, dtype=np.float32)), req, False


def to_native(S, dtype=None, host_transpose: bool = False, ctx=None):
    """A spectrogram-like array ``(..., bins, frames)``, host or device, real or complex, in any layout ->
    (DeviceArray in the kernels' native [frame][bin] "ft" layout, whether the caller owns it).

    A device array already in "ft" comes back as it is; any other goes through the transpose kernel, host arrays
    after a C-ordered upload as ``dtype``.  ``host_transpose``: reorder a host array with NumPy instead (no copy
    when its memory already is [frame][bin]) — for complex128, which the transpose kernel does not take.  Host
    arrays go to ``ctx`` (default: the default context)."""
    if not isinstance(S, nat.DeviceArray):
        ctx = ctx or nat.default_context()
        if not host_transpose:
            raw = ctx.to_device(np.ascontiguousarray(S, dtype=dtype))
            out, _ = to_native(raw)
            raw.free()
            return out, True
        view = np.swapaxes(S, -1, -2)
        mem = np.ascontiguousarray(view, dtype=dtype)
        out = nat.DeviceArray.empty(ctx, S.shape, dtype, layout="ft")
        if mem.nbytes:
            nat.check(nat.lib().b2l_h2d(ctx.handle, C.c_void_p(out.ptr), mem.ctypes.data_as(C.c_void_p), mem.nbytes))
            if mem is not view:   # a staging copy made here must outlive the upload
                ctx.synchronize()
        return out, True
    if S.layout == "ft":
        return S, False
    out = nat.DeviceArray.empty(S.ctx, S.shape, S.dtype, layout="ft")
    nat.check(nat.lib().b2l_transpose(S.ctx.handle, C.c_void_p(S.ptr), clip_count(S.shape[:-2]), S.shape[-2],
                                      S.shape[-1], S.dtype.itemsize, C.c_void_p(out.ptr)))
    return out, True


# --------------------------------------------------------------------------------------------- forward ops
_secondary = {}


def _second_context(primary):
    """A second stream (Context) on the same device, so that the H2D copy of one chunk overlaps the kernel
    and the D2H copy of the previous one (PCIe is full duplex; one stream would serialise them)."""
    ctx = _secondary.get(primary.device)
    if ctx is None:
        ctx = nat.Context(primary.device)
        _secondary[primary.device] = ctx
    return ctx


def host_chunks(n_clips: int, nbytes: int) -> int:
    """How many chunks a host batch is cut into (B2L_HOST_CHUNKS overrides; 1 disables the pipeline)."""
    env = os.environ.get("B2L_HOST_CHUNKS")
    if env:
        return max(1, min(int(env), n_clips))
    if n_clips < 8 or nbytes < (32 << 20):
        return 1
    return int(min(16, n_clips // 4))   # 16 chunks: the un-overlapped head / tail is 1/16 of the transfer


def run_forward(y, *, plan_key, plan_kw, n_frames: int, out_tail, dtype, launch, layout: str = "c",
                scratch_per_clip: int = 0):
    """Run one forward op over a signal batch ``y`` (..., n) that forward_front has accepted.

    ``nat.make_plan(ctx, plan_key, **plan_kw)`` gives the Plan; ``launch(ctx, plan, d_in, n_clips, n, d_out,
    d_scratch)`` enqueues the kernels; ``out_tail`` is the logical per-clip shape of the result in ``layout``.
    A DeviceArray ``y`` gets one launch on ``y.ctx`` and a DeviceArray result.  A host batch is validated like
    util.valid_audio and comes back as a NumPy array (pinned when large; "ft": a swapped view of [frame][bin]
    memory); large batches are cut into chunks that alternate between two streams, so that chunk i+1 uploads
    while chunk i computes and downloads."""
    n_fft, hop, center = plan_kw["n_fft"], plan_kw["hop_length"], plan_kw["center"]
    primary = context_for(y)
    lead, n = tuple(y.shape[:-1]), y.shape[-1]
    n_clips = clip_count(lead)
    plan = nat.make_plan(primary, plan_key, **plan_kw)
    assert plan.n_frames(n) == n_frames
    dtype = np.dtype(dtype)
    out_tail = tuple(out_tail)
    if isinstance(y, nat.DeviceArray):
        out = nat.DeviceArray.empty(primary, lead + out_tail, dtype, layout=layout)
        d_scr = primary.alloc(n_clips * scratch_per_clip * 4) if scratch_per_clip else 0
        launch(primary, plan, y.ptr, n_clips, n, out.ptr, d_scr)
        primary.free(d_scr)   # stream-ordered pool: the block can be handed out again without a sync
        return out
    L = nat.lib()
    flat = np.ascontiguousarray(y, dtype=np.float32).reshape(n_clips, n)
    mem_tail = out_tail[::-1] if layout == "ft" else out_tail
    per_clip_out = int(np.prod(mem_tail, dtype=np.int64))
    total_out = n_clips * per_clip_out * dtype.itemsize
    out = nat.pinned_empty((n_clips,) + mem_tail, dtype) if total_out >= (1 << 20) else \
        np.empty((n_clips,) + mem_tail, dtype)
    k = host_chunks(n_clips, flat.nbytes)
    ctxs = [primary] if k == 1 else [primary, _second_context(primary)]
    tail_begin = _uncovered_begin(n_fft, hop, center, n_frames)
    bounds = [(i * n_clips) // k for i in range(k + 1)]
    held = []
    used = []
    try:
        for i in range(k):
            lo, hi = bounds[i], bounds[i + 1]
            if hi <= lo:
                continue
            ctx = ctxs[i % len(ctxs)]
            if ctx not in used:
                nat.check(L.b2l_status_reset(ctx.handle))
                used.append(ctx)
            plan = nat.make_plan(ctx, plan_key, **plan_kw)
            m = hi - lo
            d_in = ctx.alloc(m * n * 4)
            d_out = ctx.alloc(max(m * per_clip_out * dtype.itemsize, 16))
            d_scr = ctx.alloc(m * scratch_per_clip * 4) if scratch_per_clip else 0
            held.append((ctx, d_in, d_out, d_scr))
            src = flat[lo:hi]
            nat.check(L.b2l_h2d(ctx.handle, C.c_void_p(d_in), src.ctypes.data_as(C.c_void_p), src.nbytes))
            if tail_begin < n:
                nat.check(L.b2l_scan_finite(ctx.handle, C.c_void_p(d_in), m, n, n, tail_begin))
            launch(ctx, plan, d_in, m, n, d_out, d_scr)
            dst = out[lo:hi]
            if dst.nbytes:
                nat.check(L.b2l_d2h(ctx.handle, dst.ctypes.data_as(C.c_void_p), C.c_void_p(d_out), dst.nbytes))
        flags = [status_word(ctx) for ctx in used]   # reads every stream's word: each read synchronises it
    finally:
        for ctx, d_in, d_out, d_scr in held:
            ctx.free(d_in)
            ctx.free(d_out)
            ctx.free(d_scr)
    if any(f & 1 for f in flags):
        raise ParameterError(_NOT_FINITE)
    res = out.reshape(lead + mem_tail)
    return np.swapaxes(res, -1, -2) if layout == "ft" else res
