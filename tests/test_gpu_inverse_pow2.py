"""GPU (-m gpu): the power-of-two inverse kernel (csrc/inv_kernel.cuh, launched by run_inverse in csrc/spectrum_api.cu)
at all eleven sizes n_fft = 8 ... 8192, against a float64 reference built here: scipy.fft.irfft of the complex64 input
widened to complex128, the float64 window (get_window + pad_center), a plain overlap-add, and the oracle's
window-sum-square.  The slot / piece / halo / carry schedule itself is restated for the CPU in
tests/test_inverse_gather_algorithm.py.

Most tests call b2l_istft the way core/spectrum.py::istft does (plan, reciprocal window-sum-square, device
pointers) but into an output buffer the test filled with NaN, with a row stride of its choosing: every sample
inside out_len must come back finite and within bounds, every padding sample must still be NaN.  The public istft
takes its output from the recycled device pool, where a sample the kernel forgot can hold the right value of the
previous call.  One call per group goes through lb.istft, which pins the wrapper's n_frames / out_len arithmetic.

Tolerances.
    elementwise (the project contract)   |y wss - ola| <= 1e-4 |ola| + 1e-5 max|ola of the clip| on the
                                         un-normalised overlap-add
    bit for bit                          a clip inside a batch against the same clip inverted alone (other slot
                                         cuts, same summation order), and the 16-byte gather loop against the
                                         scalar one
    norm-wise, per frame                 ||y_frame wss - w irfft(D_frame)||_2 <= C u log2(n_fft) ||w irfft(D_frame)||_2,
      (hop = n_fft, not centred)         u = 2^-24: catches a mis-rounded window or twiddle table, which passes the
                                         elementwise contract (a window table rounded to 12 mantissa bits exceeds
                                         this bound more than tenfold)

C_FRAME is the largest ratio measured by test_per_frame_norm_bound on an H100 80GB HBM3 (700 W power limit), with
about 3x headroom:
    n_fft        8     16     32     64    128    256    512   1024   2048   4096   8192
    ratio     1.37   0.99   1.50   0.38   0.49   0.26   0.88   0.68   0.57   0.75   0.27      C_FRAME = 4.5

Kernel instances (inv_inst.cu) an H100 reaches, recomputed from run_inverse with the 232 448 bytes of opt-in shared
memory the context reports (test_inverse_gather_algorithm.py::test_variants_an_h100_reaches, asserted here against
the device's own limit):
    n_fft 8 ... 512   the single instance, G = 32 frames per round
    n_fft 1024        dual halves (G = 16 each) at every hop; the 16-warp instance is never reached
    n_fft 2048        dual halves (G = 8) at every hop; the 16- and 8-warp instances are never reached
    n_fft 4096        dual halves (G = 4) for hop >= 48, 16 warps (G = 8) for hop <= 47; 8 warps never reached
    n_fft 8192        16 warps (G = 4) for hop >= 4192, 8 warps (G = 2) below — its default hop 2048 included
No hop is refused at any size.
"""
import ctypes

import numpy as np
import pytest
import scipy.fft as sf
import scipy.signal

from oracle import ref_np as O
from test_gpu_chirpz import burst, contract_close, istft_used_frames, to_device_ft
from test_inverse_gather_algorithm import H100_SMEM_OPTIN, choose_variant, slot_count, slot_length

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

SIZES = [2 << q for q in range(2, 13)]
U = 2.0 ** -24
C_FRAME = 4.5                       # norm-wise bound in units of u log2(n_fft), see the module docstring


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    return librosa_b200


@pytest.fixture(scope="module")
def smem_optin(lb):
    import torch

    return int(torch.cuda.get_device_properties(lb.default_context().device).shared_memory_per_block_optin)


# ------------------------------------------------------------------ reference
def window(name, n_fft, win_length=None):
    return O.pad_center(scipy.signal.get_window(name, win_length or n_fft, fftbins=True), n_fft)


def out_length(T, n_fft, hop, center, length):
    return int(length) if length else n_fft + hop * (T - 1) - (2 * (n_fft // 2) if center else 0)


def ref_frames(Din, n_fft, win_length=None, win="hann"):
    """w * irfft(D) in float64, [clip, frame, n_fft]."""
    return sf.irfft(Din.astype(np.complex128), n=n_fft, axis=-1) * window(win, n_fft, win_length)


def ref_ola(Din, n_fft, hop, win_length=None, center=True, length=None, win="hann"):
    """Un-normalised overlap-add of the frames istft uses, cropped like istft, and the window-sum-square it divides
    by (1 where it is tiny)."""
    T = istft_used_frames(Din.shape[-2], n_fft, hop, center, length)
    out_len = out_length(T, n_fft, hop, center, length)
    start = n_fft // 2 if center else 0
    fr = ref_frames(Din[:, :T], n_fft, win_length, win)
    buf = np.zeros((Din.shape[0], max(n_fft + hop * (T - 1), start + out_len)))
    for f in range(T):
        buf[:, f * hop:f * hop + n_fft] += fr[:, f]
    wss = O.window_sumsquare(win, T, hop_length=hop, win_length=win_length, n_fft=n_fft, dtype=np.float64)
    wss = O.fix_length(wss[start:], out_len)
    return buf[:, start:start + out_len], np.where(wss > O.tiny(wss), wss, 1.0)


def spectrum(n_clips, T, n_fft, hop, seed, win_length=None, center=True, win="hann"):
    """The float64 STFT ([clip, frame, bin]) of a -60 dB noise floor with one burst per clip, T frames a clip."""
    n = hop * (T - 1) + (0 if center else n_fft)
    y = burst(n_clips, max(n, 2), n_fft, seed).astype(np.float64)
    if center:
        y = np.pad(y, [(0, 0), (n_fft // 2, n_fft // 2)])
    y = y[:, :hop * (T - 1) + n_fft]
    frames = np.lib.stride_tricks.sliding_window_view(y, n_fft, axis=-1)[:, ::hop]
    assert frames.shape[1] == T
    return sf.rfft(frames * window(win, n_fft, win_length), axis=-1).astype(np.complex64)


# ------------------------------------------------------------------ the kernel under a NaN-filled output
def native_istft(lb, Din, n_fft, hop, win_length=None, center=True, length=None, win="hann", pad=0, offset=0):
    """b2l_istft as core/spectrum.py::istft calls it, into a NaN-filled buffer with y_stride = out_len + pad that
    starts `offset` floats into its allocation.  Din is [clip, frame, bin] complex64 on the host.  Returns the
    [clip, out_len] result after checking that it is finite and that no padding sample was touched."""
    from librosa_b200 import _native as nat, _pipeline as pl
    from librosa_b200.core import spectrum as sp

    ctx = lb.default_context()
    n_clips, T_stored = Din.shape[0], Din.shape[1]
    T = istft_used_frames(T_stored, n_fft, hop, center, length)
    out_len = out_length(T, n_fft, hop, center, length)
    stride = out_len + pad
    w, wkey = pl.resolve_window(win, win_length or n_fft, n_fft)
    plan = nat.make_plan(ctx, ("stft", n_fft, hop, bool(center), "constant", wkey), n_fft=n_fft, hop_length=hop,
                         center=center, pad_mode="constant", window=w)
    inv_ptr = sp._inv_wss(ctx, win, T, win_length or n_fft, n_fft, hop, n_fft // 2 if center else 0, out_len, wkey)
    Dd = to_device_ft(lb, Din)
    total = offset + n_clips * stride + 4
    buf = lb.DeviceArray.empty(ctx, (total,), np.float32).set(np.full(total, np.nan, dtype=np.float32))
    vp = ctypes.c_void_p
    nat.check(nat.lib().b2l_istft(ctx.handle, plan.handle, vp(Dd.ptr), n_clips, T_stored, T, vp(inv_ptr), out_len,
                                  vp(buf.ptr + 4 * offset), stride))
    host = buf.get()
    rows = host[offset:offset + n_clips * stride].reshape(n_clips, stride)
    assert np.isnan(host[:offset]).all() and np.isnan(host[offset + n_clips * stride:]).all(), "wrote outside the rows"
    assert np.isnan(rows[:, out_len:]).all(), "wrote into the row padding"
    y = rows[:, :out_len].copy()
    assert np.isfinite(y).all(), f"{int((~np.isfinite(y)).sum())} samples not written (n_fft={n_fft} hop={hop})"
    return y


def check(lb, Din, what, public=False, **kw):
    """native_istft (and the public istft when asked) against the float64 overlap-add, on the elementwise contract."""
    ola, wss = ref_ola(Din, **{k: v for k, v in kw.items() if k in ("n_fft", "hop", "win_length", "center", "length", "win")})
    y = native_istft(lb, Din, **kw)
    contract_close(y * wss, ola, what)
    if public:
        yp = lb.istft(to_device_ft(lb, Din), n_fft=kw["n_fft"], hop_length=kw["hop"], win_length=kw.get("win_length"),
                      center=kw.get("center", True), length=kw.get("length"), window=kw.get("win", "hann"))
        assert isinstance(yp, lb.DeviceArray) and yp.dtype == np.float32
        np.testing.assert_array_equal(yp.get(), y, err_msg=f"lb.istft {what}")
    return y


def variant(n_fft, hop, smem_optin):
    got = choose_variant(int(np.log2(n_fft)) - 1, hop, smem_optin)
    assert got is not None, (n_fft, hop)
    return got[:3]


# ------------------------------------------------------------------ hop sweep
def sweep_hops(n_fft):
    m4 = 3 * n_fft // 8 // 4 * 4
    if m4 < 12 or m4 & (m4 - 1) == 0:
        m4 = 12                                                   # a multiple of 4 that is no power of two
    hops = [1] if n_fft <= 256 else []
    hops += [n_fft // 16, n_fft // 8, n_fft // 4, n_fft // 4 + 1, (n_fft // 3) | 1, m4, n_fft // 2, n_fft - 4,
             n_fft - 1, n_fft, n_fft + 1, n_fft + n_fft // 3]
    return sorted({h for h in hops if h >= 1})


@pytest.mark.parametrize("n_fft", SIZES)
def test_hop_sweep(lb, n_fft):
    """Hops from 1 to above n_fft on both gather loops (16-byte and scalar; shift and division); centre on and off,
    win_length < n_fft, length absent / shorter / longer than natural (by more than a round of 32 frames, so that the
    zero-fill after the carry flush has samples to write), Hann and a window
    without zero end taps — spread over the hops."""
    for i, hop in enumerate(sweep_hops(n_fft)):
        overlap = -(-n_fft // hop)
        T = max(5, min(2 * overlap + 3, 600)) + i % 3
        center = i % 3 != 1
        win_length = n_fft - n_fft // 4 - 1 if i % 4 == 2 else None
        win = "hamming" if i % 5 == 3 else "hann"
        natural = out_length(T, n_fft, hop, center, None)
        length = [None, max(1, natural - n_fft // 2 - hop - 1), natural + 33 * hop + n_fft + 3][i % 3 if natural > 1 else 0]
        Din = spectrum(2, T, n_fft, hop, seed=n_fft + hop, win_length=win_length, center=center, win=win)
        kw = dict(n_fft=n_fft, hop=hop, win_length=win_length, center=center, length=length, win=win)
        check(lb, Din, f"istft {kw}", public=i % 4 == 0, pad=i % 2 * 3, **kw)


# ------------------------------------------------------------------ slot boundaries
def slot_batches(lb, n_fft, hop, smem_optin):
    """(n_clips, frames per clip) of batches cut into at least as many slots as there are SMs, with an odd number of
    frames per clip (coprime to 4 G) so the cuts fall at many frame offsets: one at the floor slot length 4 G, one
    where the slot length is total / (sm_count halves) rounded up."""
    sm = lb.default_context().sm_count
    _, G, halves = variant(n_fft, hop, smem_optin)
    T = 6 * G + 1
    out = []
    for factor, floor in ((1.0, True), (1.3, False)):
        n_clips = int(factor * 4 * G * sm * halves) // T
        fps = slot_length(n_clips * T, sm, halves, G)
        assert (fps == 4 * G) == floor and fps % G == 0
        slots = slot_count(n_clips * T, fps)
        assert slots > 0.8 * sm * halves                          # dual halves: more slots than SMs
        assert len({(s * fps) % T for s in range(slots)}) >= min(T, slots) // 2
        out.append((n_clips, T))
    return out


def batch_against_single_clips(lb, n_fft, hop, n_clips, T, center, seed):
    """The batch on the elementwise contract, and a handful of its clips bit for bit against the clip inverted alone
    (one or two slots instead of a cut somewhere inside)."""
    base = spectrum(7, T, n_fft, hop, seed=seed, center=center)
    scale = np.random.default_rng(seed).uniform(0.25, 4.0, n_clips).astype(np.float32)
    Din = base[np.arange(n_clips) % 7] * scale[:, None, None]
    kw = dict(n_fft=n_fft, hop=hop, center=center)
    y = check(lb, Din, f"istft n_fft={n_fft} hop={hop} clips={n_clips} T={T}", **kw)
    for c in sorted({0, 1, n_clips // 3, n_clips // 2, n_clips - 2, n_clips - 1} & set(range(n_clips))):
        np.testing.assert_array_equal(y[c], native_istft(lb, Din[c:c + 1], **kw)[0], err_msg=f"clip {c} of {n_clips}")
    return y


@pytest.mark.parametrize("n_fft", SIZES)
def test_slot_boundaries(lb, n_fft, smem_optin):
    """More slots than one wave of half-CTAs, cut at many frame offsets: halo rebuild, chunk ownership, carry."""
    for hop, center in ((max(1, n_fft // 4), True), ((n_fft // 3) | 1, False)):
        for n_clips, T in slot_batches(lb, n_fft, hop, smem_optin)[(0 if center else 1):][:1]:
            batch_against_single_clips(lb, n_fft, hop, n_clips, T, center, seed=n_fft + 1)


@pytest.mark.parametrize("n_fft", SIZES)
def test_slots_of_many_short_clips(lb, n_fft, smem_optin):
    """Clips of 1, 2 and overlap - 1 frames: a slot holds many whole clips, and a halo would reach before the clip
    start."""
    hop = max(1, n_fft // 8)
    _, G, halves = variant(n_fft, hop, smem_optin)
    for T in (1, 2, n_fft // hop - 1):
        n_clips = (4 * G * 3) // T + 5
        batch_against_single_clips(lb, n_fft, hop, n_clips, T, center=T == 2, seed=n_fft + T)


# ------------------------------------------------------------------ loud next to quiet
@pytest.mark.parametrize("n_fft", SIZES)
def test_loud_and_quiet_neighbours(lb, n_fft):
    """One clip 80 dB above its neighbours, and a loud last frame of one clip before the quiet first frame of the
    next, all inside one slot: a halo or a carry that leaked across a clip boundary would show at the quiet clip's
    own scale."""
    hop = max(1, n_fft // 4)
    Din = spectrum(5, 7, n_fft, hop, seed=n_fft + 3)
    Din[1] *= 1e4
    Din[3, -1] *= 1e4
    kw = dict(n_fft=n_fft, hop=hop)
    y = check(lb, Din, f"istft n_fft={n_fft} loud / quiet", public=True, **kw)
    for c in (0, 2, 4):
        assert np.abs(y[c]).max() < 1e-2 * np.abs(y[1]).max()
        np.testing.assert_array_equal(y[c], native_istft(lb, Din[c:c + 1], **kw)[0])


# ------------------------------------------------------------------ norm-wise bound per frame
def frame_ratio(lb, n_fft, smem_optin=H100_SMEM_OPTIN):
    """max over frames of ||y_frame wss - w irfft(D_frame)||_2 / (u ||w irfft(D_frame)||_2) with hop = n_fft and no
    centring (every output sample belongs to one frame), over enough frames to fill every group of several rounds."""
    _, G, _ = variant(n_fft, n_fft, smem_optin)
    Din = spectrum(3, 4 * G + 3, n_fft, n_fft, seed=n_fft + 5, center=False)
    y = native_istft(lb, Din, n_fft=n_fft, hop=n_fft, center=False)
    ref = ref_frames(Din, n_fft)
    w2 = window("hann", n_fft) ** 2
    got = y.reshape(ref.shape).astype(np.float64) * np.where(w2 > O.tiny(w2), w2, 1.0)
    err = np.sqrt(((got - ref) ** 2).sum(axis=-1))
    nrm = np.sqrt((ref ** 2).sum(axis=-1))
    assert (nrm > 0).all()
    return float((err / nrm).max()) / U


@pytest.mark.parametrize("n_fft", SIZES)
def test_per_frame_norm_bound(lb, n_fft, smem_optin):
    ratio = frame_ratio(lb, n_fft, smem_optin) / np.log2(n_fft)
    assert ratio <= C_FRAME, f"n_fft={n_fft}: ||err|| = {ratio:.3f} u log2(n_fft) ||frame|| (bound {C_FRAME})"


# ------------------------------------------------------------------ the two gather loops
@pytest.mark.parametrize("n_fft", SIZES)
def test_both_gather_loops_agree(lb, n_fft):
    """A 4-aligned geometry runs the 16-byte loop when the row stride and the output pointer are aligned too, and
    the scalar loop otherwise: same bits.  out_len is odd, so the 16-byte loop ends every row in its partial store.
    (n_fft = 64 has an odd frame-buffer stride and always takes the scalar loop.)"""
    for hop in sorted({max(4, n_fft // 4), 12 if n_fft <= 1024 else 3 * n_fft // 8, n_fft + 4}):
        T = 2 * (-(-n_fft // hop)) + 38
        Din = spectrum(3, T, n_fft, hop, seed=n_fft + hop + 7)
        natural = out_length(T, n_fft, hop, True, None)
        for length in (natural - 5, natural + n_fft + 3):
            pad = -length % 4
            assert pad                                            # the row ends inside a 16-byte item
            kw = dict(n_fft=n_fft, hop=hop, length=length)
            vec = check(lb, Din, f"16-byte loop {kw}", pad=pad, **kw)
            for how in (dict(pad=0), dict(pad=pad + 4), dict(pad=pad, offset=1)):
                np.testing.assert_array_equal(native_istft(lb, Din, **kw, **how), vec, err_msg=f"{kw} {how}")


# ------------------------------------------------------------------ CTA variants
VARIANT_CASES = [(4096, 16, (16, 8, 1)), (4096, 1024, (116, 4, 2)), (8192, 2048, (8, 2, 1)), (8192, 6144, (16, 4, 1))]


def test_variant_arithmetic_holds_on_this_device(smem_optin):
    assert smem_optin == H100_SMEM_OPTIN
    for n_fft, hop, want in VARIANT_CASES:
        assert variant(n_fft, hop, smem_optin) == want


@pytest.mark.parametrize("n_fft,hop,want", VARIANT_CASES)
def test_variants_on_slot_boundaries(lb, n_fft, hop, want, smem_optin):
    """Both sides of the dual / 16-warp switch of n_fft 4096 and of the 16- / 8-warp switch of n_fft 8192, each on a
    batch that fills every slot."""
    n_clips, T = slot_batches(lb, n_fft, hop, smem_optin)[0]
    batch_against_single_clips(lb, n_fft, hop, n_clips, T, center=True, seed=hop)


@pytest.mark.parametrize("n_fft", SIZES)
def test_no_hop_is_refused(lb, n_fft):
    """hop 1 (the largest carry) and hop 3 n_fft (no carry at all)."""
    for hop in (1, 3 * n_fft):
        Din = spectrum(2, 5, n_fft, hop, seed=n_fft + hop)
        kw = dict(n_fft=n_fft, hop=hop)
        check(lb, Din, f"istft {kw}", **kw)


# ------------------------------------------------------------------ irfft semantics
@pytest.mark.parametrize("n_fft", SIZES)
def test_imaginary_dc_and_nyquist_are_ignored(lb, n_fft):
    rng = np.random.default_rng(n_fft)
    hop = max(1, n_fft // 4)
    Din = spectrum(2, 9, n_fft, hop, seed=n_fft + 11)
    scale = float(np.abs(Din).max())
    for k in (0, -1):
        Din[..., k] += (1j * scale * rng.uniform(0.5, 1.0, Din.shape[:-1]) * rng.choice([-1, 1], Din.shape[:-1])).astype(np.complex64)
    kw = dict(n_fft=n_fft, hop=hop)
    clean = Din.copy()
    clean[..., 0].imag = 0
    clean[..., -1].imag = 0
    np.testing.assert_array_equal(check(lb, Din, f"istft n_fft={n_fft} Im DC / Nyquist", public=True, **kw),
                                  native_istft(lb, clean, **kw))


@pytest.mark.parametrize("n_fft", SIZES)
def test_unused_frames_are_not_read(lb, n_fft):
    """length makes istft use fewer frames than the matrix stores: NaN in the unused ones changes nothing."""
    hop = max(1, n_fft // 4)
    T_stored, T = 40, 29
    Din = spectrum(3, T_stored, n_fft, hop, seed=n_fft + 13)
    length = hop * T - 2 * (n_fft // 2)
    assert istft_used_frames(T_stored, n_fft, hop, True, length) == T
    kw = dict(n_fft=n_fft, hop=hop, length=length)
    y = check(lb, Din, f"istft {kw}", **kw)
    Din[:, T:] = np.nan
    np.testing.assert_array_equal(native_istft(lb, Din, **kw), y)
    yp = lb.istft(to_device_ft(lb, Din), n_fft=n_fft, hop_length=hop, length=length)
    np.testing.assert_array_equal(yp.get(), y)


# ------------------------------------------------------------------ device-resident consumers
@pytest.mark.parametrize("n_fft", [64, 4096])
def test_consumers(lb, n_fft):
    """griffinlim and effects.hpss hand the kernel DeviceArrays in the native layout; tolerances of test_gpu_parity /
    test_gpu_features."""
    import signals

    hop = n_fft // 4
    y = signals.make("B", (2, 12 * n_fft + 1000), seed=n_fft)
    S = np.abs(O.stft(y[0], n_fft=n_fft, hop_length=hop))
    got = lb.griffinlim(S, n_iter=2, init=None, n_fft=n_fft, hop_length=hop)
    want = O.griffinlim(S, n_iter=2, init=None, n_fft=n_fft, hop_length=hop)
    assert got.shape == want.shape and got.dtype == want.dtype
    np.testing.assert_allclose(got, want, rtol=0, atol=2e-3 * float(np.abs(want).max()))
    dev = lb.effects.hpss(lb.to_device(y), n_fft=n_fft, hop_length=hop)
    ref = O.effects_hpss(y, n_fft=n_fft, hop_length=hop)
    for a, b in zip(dev, ref):
        assert isinstance(a, lb.DeviceArray)
        np.testing.assert_allclose(a.get(), b, rtol=1e-4, atol=2e-5 * float(np.abs(b).max()))
