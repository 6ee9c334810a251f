"""GPU (-m gpu): the fused mel / MFCC front end — fwd_kernel in MODE_MEL (csrc/fwd_kernel.cuh) for the powers of two,
mr_kernel<2, G> (csrc/mr_kernel.cuh) for the mixed-radix sizes, then dct_clamp4_kernel<KS> / dct_generic_kernel
(csrc/aux_kernels.cuh) — at every kernel instance, tile geometry and clip boundary, against a float64 reference built
here: the float32 samples widened, np.pad, the float64 window (get_window + pad_center), scipy.fft.rfft, |X|**power,
the library's float32 mel basis widened, 10 log10(max(amin, .)), the per-clip clamp at max - 80 dB and SciPy's DCT.
The host side (instance choice, MelRow table, DCT choice) is restated in tests/test_mel_front_end_algorithm.py.

Most tests call b2l_melspectrogram / b2l_mfcc the way feature/spectral.py does (same plans), but into NaN-filled
outputs with guard words on both sides and, for b2l_mfcc, a NaN-filled log-mel scratch the test reads back: every
valid value must come back finite, every guard word and every padding frame of the tiled scratch must still be NaN.
Each instance first runs on NaN audio through the public API (which raises ParameterError), so shared memory holds
NaN when the checked call starts, and a read of a word the tile did not write shows up.  One call per group goes
through the public function and must equal the native call bit for bit.

Tolerances.
    mel, elementwise (the contract)   |mel - mel64| <= 1e-4 |mel64| + 1e-6 max(mel64 of the clip)
    mel, norm-wise per frame          ||mel - mel64||_2 <= C_MEL u log2(n_fft) ||mel64||_2 over the mel axis, u = 2^-24;
                                      weights rounded to 12 mantissa bits exceed it (and pass the elementwise contract
                                      in most bins)
    mfcc, elementwise (the contract)  |mfcc - mfcc64| <= 1e-4 |mfcc64| + 1e-3
    clamp + DCT, isolated             the float64 DCT (the plan's float32 DCT rows widened) of max(L, max_clip(L) - 80)
                                      computed in float32 from the kernel's own log-mel L: |err| <= n_mels u (|D| |X|)
    dB epilogue                       |L - 10 log10(max(amin, mel))| <= DB_ABS + DB_REL |L|, mel the kernel's own values
                                      (2e-6 + 2^-21 |L|: MUFU.LG2 is about 2 ulp of the result; measured on the H100 at
                                      most 1.7e-5 dB, near the -100 dB floor, and 0.69 of 1e-6 + 2^-22 |L|)
    bit for bit                       a clip in a batch against the clip alone, input one float off alignment against
                                      aligned input, a host batch against a DeviceArray batch

C_MEL is the largest ratio measured by test_per_frame_norm_bound and test_mixed_radix_sizes on an H100 80GB HBM3 (700 W
power limit), with about 3x headroom:
    n_fft        8     16     32     64    128    256    512   1024   2048   4096   8192   mixed radix (96 sizes)
    ratio     1.22   1.57   1.10   0.90   0.72   0.49   0.42   0.39   0.42   0.26   0.20   at most 1.05 (n_fft 40)
                                                                                                    C_MEL = 5
"""
import ctypes
from functools import lru_cache

import numpy as np
import pytest
import scipy.fft as sf

from test_gpu_chirpz import burst, contract_close
from test_gpu_inverse_pow2 import window
from test_mel_front_end_algorithm import H100_MEL_VARIANTS, forward_choice, mel_basis, mr_sizes

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

SIZES = [2 << q for q in range(2, 13)]
U = 2.0 ** -24
C_MEL = 5.0                          # norm-wise bound in units of u log2(n_fft), see the module docstring
DB_ABS, DB_REL = 2e-6, 2.0 ** -21    # dB epilogue, see the module docstring
AMIN = float(np.float32(1e-10))
GUARD = 37                           # NaN words before and after every output


# ------------------------------------------------------------------ signals and the float64 reference
def n_samples(T, n_fft, hop, center):
    """A signal length that gives exactly T frames; a multiple of 4 when the hop is, so that such clips qualify for
    the bulk copy of fwd_kernel (see bulk_copy) and the vector loads of mr_kernel."""
    n = hop * (T - 1) + (hop - 1) // 2 // 4 * 4 + (0 if center else n_fft)
    assert n >= 1 and 1 + (n + (2 * (n_fft // 2) if center else 0) - n_fft) // hop == T, (T, n_fft, hop)
    return n


def signals(n_clips, n, n_fft, seed):
    """-60 dB noise with one unit-level burst per clip (test_gpu_chirpz.burst), float32."""
    return burst(n_clips, n, n_fft, seed)


def ref_power(y, n_fft, hop, win_length=None, center=True, pad_mode="constant", power=2.0):
    """|rfft(frame * window)|**power in float64, [clip, frame, bin]."""
    y = np.asarray(y, dtype=np.float64)
    if center:
        y = np.pad(y, [(0, 0), (n_fft // 2, n_fft // 2)], mode=pad_mode)
    frames = np.lib.stride_tricks.sliding_window_view(y, n_fft, axis=-1)[:, ::hop]
    return np.abs(sf.rfft(frames * window("hann", n_fft, win_length), axis=-1)) ** power


def ref_mel(P, basis):
    """[clip, mel, frame] float64."""
    return np.ascontiguousarray(np.matmul(P, np.asarray(basis, dtype=np.float64).T).transpose(0, 2, 1))


def ref_db(mel):
    return 10.0 * np.log10(np.maximum(AMIN, mel))


@lru_cache(maxsize=None)
def tile_frames(n_fft, hop, n_mels=128):
    """FT of the fwd_kernel instance MODE_MEL runs at this hop (sr 22 050), from the restated run_forward."""
    return forward_choice(n_fft, hop, mel_basis(22050, n_fft, n_mels))[1]


def bulk_copy(n_fft, hop, y_stride, offset):
    """run_forward's tma_ok (spectrum_api.cu) for a clip `offset` floats past a 16-byte aligned allocation: base, row
    stride and staged span (FT - 1) hop + n_fft all 16-byte aligned.  Interior tiles then stage by TMA bulk copy
    (TILE_TMA; edge tiles TILE_TMA_ZERO or the gather); otherwise every tile takes the per-sample gather."""
    return offset % 4 == 0 and y_stride % 4 == 0 and ((tile_frames(n_fft, hop) - 1) * hop + n_fft) % 4 == 0


def vector_loads(n_fft, hop, y_stride, offset):
    """mr_kernel's vec_ok (8-byte aligned base, even row stride) and even frame starts s0 = frame hop - n_fft / 2:
    interior frames then load sample pairs as float2; otherwise every frame takes the scalar np.pad index map."""
    return offset % 2 == 0 and y_stride % 2 == 0 and hop % 2 == 0 and (n_fft // 2) % 2 == 0


def norm_ratio(got, ref):
    """max over frames of ||got - ref||_2 / (u ||ref||_2) along the mel axis; frames with ref == 0 must be exact."""
    err = np.sqrt(((got.astype(np.float64) - ref) ** 2).sum(axis=1))
    nrm = np.sqrt((ref ** 2).sum(axis=1))
    assert not err[nrm == 0].any(), "a silent frame is not exactly zero"
    return float((err[nrm > 0] / nrm[nrm > 0]).max(initial=0.0)) / U


def mel_close(got, ref, n_fft, what):
    """The mel checks: the elementwise contract and the per-frame norm-wise bound."""
    contract_close(got, ref, what, rtol=1e-4, atol_rel=1e-6)
    ratio = norm_ratio(got, ref) / np.log2(n_fft)
    assert ratio <= C_MEL, f"{what}: ||err|| = {ratio:.3f} u log2(n_fft) ||mel|| (bound {C_MEL})"
    return ratio


def mfcc_close(got, ref, what):
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got.astype(np.float64) - ref)
    bad = ~(err <= 1e-4 * np.abs(ref) + 1e-3)
    assert not bad.any(), f"{what}: {int(bad.sum())} coefficients, max |err| = {float(err.max()):.3e}"


# ------------------------------------------------------------------ the kernels under NaN-filled outputs
@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    return librosa_b200


def mel_kwargs(kw):
    return {k: kw[k] for k in ("n_mels", "fmin", "fmax", "htk", "norm") if k in kw}


def make_plan(lb, n_fft, hop, kw, n_mfcc=0):
    """The plan feature/spectral.py makes for melspectrogram (n_mfcc 0) or mfcc, and its float32 mel basis and DCT
    rows."""
    from librosa_b200 import _native as nat, _pipeline as pl
    from librosa_b200.feature import spectral as S

    ctx = lb.default_context()
    center = kw.get("center", True)
    w, wkey = pl.resolve_window("hann", kw.get("win_length") or n_fft, n_fft)
    mode = kw.get("pad_mode", "constant") if center else "constant"
    power = float(kw.get("power", 2.0))
    mk = mel_kwargs(kw)
    if n_mfcc:
        mk["norm"] = kw.get("norm", "slaney")
    basis, bkey = pl.mel_basis(kw.get("sr", 22050), n_fft, mk)
    plan_kw = dict(n_fft=n_fft, hop_length=hop, center=center, pad_mode=mode, window=w, mel_basis=basis, power=power)
    if not n_mfcc:
        return nat.make_plan(ctx, ("mel", n_fft, hop, bool(center), mode, wkey, bkey, power), **plan_kw), basis, None
    dct = S._dct_basis(basis.shape[0], n_mfcc, 2, "ortho", kw.get("lifter", 0))
    plan = nat.make_plan(ctx, ("mfcc", n_fft, hop, bool(center), mode, wkey, bkey, power, pl.digest(dct)),
                         dct_basis=dct, amin=1e-10, ref_value=1.0, top_db=80.0, **plan_kw)
    return plan, basis, dct


def nan_buffer(lb, words):
    return lb.DeviceArray.empty(lb.default_context(), (words,), np.float32).set(np.full(words, np.nan, np.float32))


def device_input(lb, y, offset):
    flat = np.concatenate([np.zeros(offset, np.float32), y.ravel(), np.zeros(4, np.float32)])
    return lb.DeviceArray.empty(lb.default_context(), flat.shape, np.float32).set(flat)


def unguard(host, what, guard=GUARD):
    assert np.isnan(host[:guard]).all() and np.isnan(host[-guard:]).all(), f"{what}: wrote outside the output"
    return host[guard:-guard]


def native(lb, y, n_fft, hop, n_mfcc=0, offset=0, guard=GUARD, **kw):
    """b2l_melspectrogram (n_mfcc 0) or b2l_mfcc on the float32 batch y [clip, n], the input `offset` floats into its
    allocation, the outputs `guard` floats into theirs (the default 37 leaves them off 16-byte alignment).  Returns
    mel [clip, mel, frame], or (mfcc [clip, k, frame], log-mel [clip, mel, frame])."""
    from librosa_b200 import _native as nat, _pipeline as pl

    ctx = lb.default_context()
    vp = ctypes.c_void_p
    plan, basis, dct = make_plan(lb, n_fft, hop, kw, n_mfcc)
    n_mfcc = dct.shape[0] if n_mfcc else 0                              # at most n_mels coefficients
    n_clips, n = y.shape
    T = plan.n_frames(n)
    nm = basis.shape[0]
    what = f"n_fft={n_fft} hop={hop} clips={n_clips} T={T} {kw}"
    din = device_input(lb, y, offset)
    nat.check(nat.lib().b2l_status_reset(ctx.handle))
    blocks = (T + 63) // 64
    if not n_mfcc:
        out = nan_buffer(lb, n_clips * nm * T + 2 * guard)
        nat.check(nat.lib().b2l_melspectrogram(ctx.handle, plan.handle, vp(din.ptr + 4 * offset), n_clips, n, n,
                                               vp(out.ptr + 4 * guard)))
        res = unguard(out.get(), what, guard).reshape(n_clips, nm, T)
        out.free()
    else:
        out = nan_buffer(lb, n_clips * n_mfcc * T + 2 * guard)
        scr = nan_buffer(lb, n_clips * nm * blocks * 64 + 2 * guard)
        nat.check(nat.lib().b2l_mfcc(ctx.handle, plan.handle, vp(din.ptr + 4 * offset), n_clips, n, n,
                                     vp(out.ptr + 4 * guard), vp(scr.ptr + 4 * guard)))
        coef = unguard(out.get(), what, guard).reshape(n_clips, n_mfcc, T)
        s = unguard(scr.get(), what, guard)
        if n_fft & (n_fft - 1) == 0:      # tiled scratch [clip][64-frame block][mel][64]
            tiles = s.reshape(n_clips, blocks, nm, 64)
            assert np.isnan(tiles[:, -1, :, T - 64 * (blocks - 1):]).all(), f"{what}: wrote a padding frame"
            L = tiles.transpose(0, 2, 1, 3).reshape(n_clips, nm, blocks * 64)[..., :T]
        else:                             # mixed radix: [clip][mel][frame]
            assert np.isnan(s[n_clips * nm * T:]).all(), f"{what}: wrote past the log-mel rows"
            L = s[:n_clips * nm * T].reshape(n_clips, nm, T)
        assert np.isfinite(L).all(), f"{what}: {int((~np.isfinite(L)).sum())} log-mel values not written"
        res = (coef, np.ascontiguousarray(L))
        out.free()
        scr.free()
    din.free()
    assert not pl.status_word(ctx) & nat.STATUS_NOT_FINITE_SAMPLE, f"{what}: finite input flagged"
    first = res if not n_mfcc else res[0]
    assert np.isfinite(first).all(), f"{what}: {int((~np.isfinite(first)).sum())} values not written"
    return res


def public_kwargs(n_fft, hop, kw):
    out = dict(sr=kw.get("sr", 22050), n_fft=n_fft, hop_length=hop)
    out.update({k: v for k, v in kw.items() if k in ("center", "pad_mode", "win_length", "power", "n_mels", "fmin",
                                                       "fmax", "htk")})
    return out


def poison(lb, y_shape, n_fft, hop, n_mfcc=0, **kw):
    """The same instance on NaN audio through the public API: raises, and leaves NaN in shared memory."""
    from librosa_b200.util.exceptions import ParameterError

    nan = np.full(y_shape, np.nan, np.float32)
    pk = public_kwargs(n_fft, hop, kw)
    with pytest.raises(ParameterError):
        if n_mfcc:
            lb.feature.mfcc(y=nan, n_mfcc=n_mfcc, mel_norm=kw.get("norm", "slaney"), **pk)
        else:
            lb.feature.melspectrogram(y=nan, norm=kw.get("norm", "slaney"), **pk)


def check_mel(lb, y, n_fft, hop, public=False, **kw):
    """native melspectrogram after a poisoning call, against the float64 reference; returns (mel, ratio)."""
    poison(lb, y.shape, n_fft, hop, **kw)
    mel = native(lb, y, n_fft, hop, **kw)
    basis = make_plan(lb, n_fft, hop, kw)[1]
    P = ref_power(y, n_fft, hop, kw.get("win_length"), kw.get("center", True), kw.get("pad_mode", "constant"),
                  kw.get("power", 2.0))
    ratio = mel_close(mel, ref_mel(P, basis), n_fft, f"mel n_fft={n_fft} hop={hop} {kw}")
    if public:
        got = lb.feature.melspectrogram(y=lb.to_device(y), norm=kw.get("norm", "slaney"), **public_kwargs(n_fft, hop, kw))
        np.testing.assert_array_equal(got.get(), mel, err_msg=f"public melspectrogram n_fft={n_fft} hop={hop}")
    return mel, ratio


def check_mfcc(lb, y, n_fft, hop, n_mfcc=20, public=False, **kw):
    """native mfcc after a poisoning call: the log-mel scratch against the kernel's own mel values (dB epilogue), the
    clamp + DCT against the float64 DCT of the clamped scratch, and the result against the full float64 reference."""
    poison(lb, y.shape, n_fft, hop, n_mfcc, **kw)
    coef, L = native(lb, y, n_fft, hop, n_mfcc=n_mfcc, **kw)
    _, basis, dct = make_plan(lb, n_fft, hop, kw, n_mfcc)
    what = f"mfcc n_fft={n_fft} hop={hop} clips={y.shape[0]} {kw}"
    # dB epilogue: the same instance's mel values (melspectrogram plan with the same basis and tile geometry)
    mel = native(lb, y, n_fft, hop, **kw)
    err = np.abs(L.astype(np.float64) - ref_db(mel.astype(np.float64)))
    assert (err <= DB_ABS + DB_REL * np.abs(L)).all(), f"{what}: dB epilogue off by {float(err.max()):.3e} dB"
    # clamp + DCT from the kernel's own log-mel
    floor = L.max(axis=(1, 2)) - np.float32(80.0)
    X = np.maximum(L, floor[:, None, None]).astype(np.float64)
    D = dct.astype(np.float64)
    want = np.einsum("km,cmt->ckt", D, X)
    bound = 1.01 * basis.shape[0] * U * np.einsum("km,cmt->ckt", np.abs(D), np.abs(X))
    bad = np.abs(coef - want) > bound
    assert not bad.any(), f"{what}: clamp + DCT, {int(bad.sum())} coefficients off"
    # the whole chain against float64
    P = ref_power(y, n_fft, hop, kw.get("win_length"), kw.get("center", True), kw.get("pad_mode", "constant"),
                  kw.get("power", 2.0))
    import scipy.fft

    mel64 = ref_mel(P, basis)
    L64 = ref_db(mel64)
    L64 = np.maximum(L64, L64.max(axis=(1, 2), keepdims=True) - 80.0)
    ref = scipy.fft.dct(L64, axis=-2, type=2, norm="ortho")[:, :n_mfcc]
    mfcc_close(coef, ref, what)
    if public:
        got = lb.feature.mfcc(y=lb.to_device(y), n_mfcc=n_mfcc, mel_norm=kw.get("norm", "slaney"),
                              **public_kwargs(n_fft, hop, kw))
        np.testing.assert_array_equal(got.get(), coef, err_msg=what)
    return coef, L


# ------------------------------------------------------------------ every instance of the power-of-two kernel
def variant_cases():
    """(n_fft, hop, FT) at the first and last hop of every instance window (sr 22 050, 128 mels)."""
    out = []
    for n_fft, (runs, _) in H100_MEL_VARIANTS.items():
        for first, last, v, ft in runs:
            for hop in sorted({first, last, n_fft // 4} & set(range(first, last + 1))):
                out.append((n_fft, hop, ft))
    return out


@pytest.mark.parametrize("n_fft,hop,ft", variant_cases())
def test_every_instance_window(lb, n_fft, hop, ft):
    """Two clips of 2 FT + 1 frames (the last tile holds one frame) at the hop; the public call once per size."""
    T = 2 * ft + 1
    y = signals(2, n_samples(T, n_fft, hop, True), n_fft, seed=n_fft + hop)
    check_mel(lb, y, n_fft, hop, public=hop == n_fft // 4)


@pytest.mark.parametrize("n_fft", SIZES)
def test_first_refused_hop(lb, n_fft):
    """The refusal stays where it is: the first hop past the last instance window raises UnsupportedOnGPU."""
    from librosa_b200 import _native as nat

    stop = H100_MEL_VARIANTS[n_fft][1]
    y = signals(1, n_samples(3, n_fft, stop, True), n_fft, seed=1)
    with pytest.raises(nat.UnsupportedOnGPU):
        lb.feature.melspectrogram(y=lb.to_device(y), sr=22050, n_fft=n_fft, hop_length=stop)


@pytest.mark.parametrize("n_fft", SIZES)
def test_per_frame_norm_bound(lb, n_fft):
    """Every size at its default hop, with frames of very different level in one tile; records the ratio."""
    hop = n_fft // 4
    ft = tile_frames(n_fft, hop)
    y = signals(3, n_samples(3 * ft + 1, n_fft, hop, True), n_fft, seed=n_fft + 5)
    _, ratio = check_mel(lb, y, n_fft, hop)
    print(f"RATIO pow2 n_fft={n_fft} {ratio:.3f}")


# ------------------------------------------------------------------ the mixed-radix sizes
@pytest.mark.parametrize("n_fft", mr_sizes())
def test_mixed_radix_sizes(lb, n_fft):
    """mr_kernel<2, 16> (n_fft <= 1024) and <2, 32>: three clips whose frame count is odd, so the two lane groups of a
    warp sit in different clips at some boundaries."""
    hop = n_fft // 4 + (n_fft // 4) % 2 + 1
    n_mels = 128 if n_fft >= 256 else 40
    y = signals(3, n_samples(37, n_fft, hop, True), n_fft, seed=n_fft)
    _, ratio = check_mel(lb, y, n_fft, hop, n_mels=n_mels, public=n_fft in (400, 2400))
    print(f"RATIO mr n_fft={n_fft} {ratio:.3f}")


# ------------------------------------------------------------------ frame counts, pads, windows, powers
FRAME_COUNT_SIZES = [64, 1024, 2048, 4096, 8192]


@pytest.mark.parametrize("n_fft", FRAME_COUNT_SIZES)
def test_frame_counts(lb, n_fft):
    """T = 1, T == 1 mod FT, and 63 ... 129 around the 64-frame blocks of the tiled scratch; mel and mfcc.  The public
    functions once each, bit for bit against the native calls."""
    hop = n_fft // 4
    ft = tile_frames(n_fft, hop)
    for T in sorted({1, ft + 1, 3 * ft + 1, 63, 64, 65, 127, 128, 129}):
        y = signals(2, n_samples(T, n_fft, hop, True), n_fft, seed=n_fft + T)
        check_mel(lb, y, n_fft, hop, public=T == 1)
        check_mfcc(lb, y, n_fft, hop, n_mfcc=13, public=T == 65)


GEOMETRIES = [dict(pad_mode="reflect"), dict(pad_mode="edge"), dict(pad_mode="symmetric"),
              dict(pad_mode="linear_ramp"), dict(center=False), dict(win_length=None, power=1.0),
              dict(power=1.5, pad_mode="reflect"), dict(htk=True, fmin=300.0, fmax=4000.0, norm=None)]


@pytest.mark.parametrize("n_fft", [16, 256, 512, 2048, 8192, 400, 2400])
def test_pads_windows_powers(lb, n_fft):
    """Every pad mode, center=False, win_length < n_fft, power 1 / 1.5 (and 2), band limits with empty rows; each
    geometry also through the public melspectrogram, bit for bit, which pins its argument mapping."""
    hop = n_fft // 4
    for i, g in enumerate(GEOMETRIES):
        kw = dict(g)
        if i % 2:
            kw["win_length"] = n_fft - n_fft // 4 - 1
        center = kw.get("center", True)
        y = signals(2, n_samples(33 + i, n_fft, hop, center), n_fft, seed=n_fft + i)
        check_mel(lb, y, n_fft, hop, public=True, n_mels=64 if n_fft >= 128 else 16, **kw)


# ------------------------------------------------------------------ batches that walk across clips
def clamp_batch(n_clips, T, n_fft, hop, seed):
    """Quiet clips (a short loud head, then digital silence: more than 80 dB of range, so the clamp bites),
    neighbours 40 dB louder, and clips whose loudest frame is the last one (a loud click at the end, in the last
    tile)."""
    n = n_samples(T, n_fft, hop, True)
    y = signals(n_clips, n, n_fft, seed)
    rng = np.random.default_rng(seed)
    for c in range(n_clips):
        kind = c % 3
        if kind == 0:
            y[c] = 0.0
            y[c, :max(1, hop // 2)] = (4.0 * rng.standard_normal(max(1, hop // 2))).astype(np.float32)
        elif kind == 1:
            y[c] *= 100.0
        else:
            y[c] *= 0.1
            k = max(2, min(n, n_fft // 16))
            y[c, n - k:] += (4.0 * rng.standard_normal(k)).astype(np.float32)
    return y


@pytest.mark.parametrize("n_fft", [64, 512, 1024, 2048, 4096, 8192, 400, 2400])
def test_batches_across_clips(lb, n_fft):
    """More tiles (frames) than the grid holds, T odd: the tile walk and the lane groups cross clips.  mfcc: the
    per-clip maximum and clamp isolated against the kernel's own log-mel; a handful of clips bit for bit against
    the clip alone."""
    pow2 = n_fft & (n_fft - 1) == 0
    hop = n_fft // 4
    sm = lb.default_context().sm_count
    if pow2:                                      # 3 tiles a clip, about three times the tiles of one wave
        ft = tile_frames(n_fft, hop)
        T = 2 * ft + 1
        n_clips = (3 * sm * 2) // 3
    else:                                         # 65 frames a clip, several times the frames of one wave
        T = 65
        n_clips = (3 * sm * 2 * 32) // 33
    n_clips = min(n_clips, 300)
    y = clamp_batch(n_clips, T, n_fft, hop, seed=n_fft)
    mel, _ = check_mel(lb, y, n_fft, hop)
    coef, L = check_mfcc(lb, y, n_fft, hop, n_mfcc=20, public=True)
    rng = L.max(axis=(1, 2)) - L.min(axis=(1, 2))
    assert (rng[0::3] > 80.0).all(), "the quiet clips must exceed the clamp range"
    last = L.max(axis=1).argmax(axis=-1)
    assert (last[2::3] == T - 1).all(), "the clicked clips must peak in their last frame"
    for c in sorted({0, 1, 2, n_clips // 2, n_clips - 2, n_clips - 1}):
        np.testing.assert_array_equal(native(lb, y[c:c + 1], n_fft, hop)[0], mel[c], err_msg=f"mel clip {c}")
        one, _ = native(lb, y[c:c + 1], n_fft, hop, n_mfcc=20)
        np.testing.assert_array_equal(one[0], coef[c], err_msg=f"mfcc clip {c}")


# ------------------------------------------------------------------ bit for bit across input paths
@pytest.mark.parametrize("n_fft", [64, 1024, 2048, 8192, 400, 2400])
def test_input_paths_agree(lb, n_fft):
    """The fast input path against the fallback, bit for bit.  Baseline: the clip at the start of its allocation with
    a row stride that is a multiple of 4 and hop % 4 == 0, so tiles stage by bulk copy (power of two) and interior
    frames load sample pairs (mixed radix).  Against it: the same clips one float further on (per-sample gather and
    scalar loads), four floats further on (aligned again), and a host batch through the public API (staged
    into an aligned buffer of the same stride: the fast path once more).  mfcc adds a scratch and output off 16-byte
    alignment (4-byte tile loads in dct_clamp4_kernel) against aligned ones (16-byte loads)."""
    pow2 = n_fft & (n_fft - 1) == 0
    hop = n_fft // 4
    T = 3 * tile_frames(n_fft, hop) + 2 if pow2 else 40                # interior tiles as well as edge tiles
    n = n_samples(T, n_fft, hop, True)
    fast = bulk_copy if pow2 else vector_loads
    assert fast(n_fft, hop, n, 0) and fast(n_fft, hop, n, 4) and not fast(n_fft, hop, n, 1)
    y = signals(3, n, n_fft, seed=n_fft + 17)
    mel = native(lb, y, n_fft, hop)
    np.testing.assert_array_equal(native(lb, y, n_fft, hop, offset=1), mel)
    np.testing.assert_array_equal(native(lb, y, n_fft, hop, offset=4), mel)
    host = lb.feature.melspectrogram(y=y, sr=22050, n_fft=n_fft, hop_length=hop)
    np.testing.assert_array_equal(host, mel)
    coef, L = native(lb, y, n_fft, hop, n_mfcc=20)
    np.testing.assert_array_equal(native(lb, y, n_fft, hop, n_mfcc=20, offset=1)[0], coef)
    aligned = native(lb, y, n_fft, hop, n_mfcc=20, guard=36)          # 16-byte loads of the log-mel tiles
    np.testing.assert_array_equal(aligned[0], coef)
    np.testing.assert_array_equal(aligned[1], L)
    np.testing.assert_array_equal(lb.feature.mfcc(y=y, sr=22050, n_fft=n_fft, hop_length=hop, n_mfcc=20), coef)


# ------------------------------------------------------------------ the DCT kernels
@pytest.mark.parametrize("n_fft,n_mels,n_mfcc,kind", [
    (2048, 128, 20, "ks2"), (512, 13, 20, "ks1"), (1024, 128, 100, "ks1"), (4096, 40, 13, "ks2"),
    (2400, 400, 20, "generic"), (400, 13, 20, "ks1"), (1200, 128, 40, "ks2"),
])
def test_dct_kernels(lb, n_fft, n_mels, n_mfcc, kind):
    """dct_clamp4_kernel with KS = 2 and 1 on both paths, dct_generic_kernel on the mixed-radix path."""
    from test_mel_front_end_algorithm import dct_choice

    assert dct_choice(n_mels, min(n_mfcc, n_mels), n_fft & (n_fft - 1) == 0) == kind
    hop = n_fft // 4
    y = clamp_batch(5, 131, n_fft, hop, seed=n_fft + n_mels)
    check_mfcc(lb, y, n_fft, hop, n_mfcc=n_mfcc, n_mels=n_mels, public=kind == "generic")


def test_tiled_dct_refusal(lb):
    """n_mels too large for the tiled scratch of the power-of-two path is refused, not truncated."""
    from librosa_b200 import _native as nat

    y = signals(1, 8192, 4096, seed=3)
    with pytest.raises(nat.UnsupportedOnGPU, match="n_mels=512 is too large for the fused mfcc path"):
        lb.feature.mfcc(y=lb.to_device(y), sr=22050, n_fft=4096, hop_length=1024, n_mels=512)
