"""GPU (-m gpu): the float32 chirp-z kernels (csrc/czt_kernel.cuh: czt_kernel, czt_inv_kernel) at every transform
size P = 32 ... 4096 they are instantiated for, forward and inverse, against a float64 reference built here: np.pad
of the signal, framing, the float64 window (scipy.signal.get_window, centred to n_fft) and scipy.fft.rfft / irfft in
float64.  Inputs go in as DeviceArrays, so a routing change cannot move a size onto the FP64 kernels unnoticed.
The algorithm itself is restated in float64 for all 1 962 chirp-z frame lengths in tests/test_chirpz_algorithm.py.

Engine configuration per instance (czt_inst.cu, HostFftCfg::czt_nw): TPF = P/32 threads per frame pair and
G = 32 * NW / TPF pairs per CTA step, with G = 32 for P <= 512 and 16, 8, 4 for P = 1024, 2048, 4096.

Tolerances.
    elementwise (the project contract)   |X - X_ref| <= 1e-4 |X_ref| + 1e-5 max|X_ref of the clip|; istft on the
                                         un-normalised overlap-add (y * window-sum-square, as in test_gpu_parity)
    norm-wise, per frame pair A, B       ||X - X_ref||_2 <= C u log2(P) max(||X_ref,A||_2, ||X_ref,B||_2),
      (frames 2j, 2j+1 of a clip)        u = 2^-24; the inverse on the window-weighted frames (hop = n_fft, so
                                         every output sample belongs to one frame)
The norm-wise bound is what catches a bad table or a lost bit: both frames of a pair share one transform, so the
error of a frame scales with the louder partner, and a FFT_P(h)/P table rounded to 14 mantissa bits passes the
elementwise contract in most bins but exceeds this bound more than tenfold.  The istft outputs cover every sample the
frames came from (a centred istft of natural length drops the signal's tail, and a loud frame there would carry its
round-off into the kept samples of a quiet clip).

C is the largest ratio ||err|| / (u log2(P) max(||A||, ||B||)) measured over this file's cases on an H100 80GB HBM3
(700 W power limit), with about 3.5x headroom, one constant per direction:
    P           32     64    128    256    512   1024   2048   4096
    forward   0.87   0.83   0.60   0.58   0.54   0.47   0.47   0.42      C_FWD = 3
    inverse   5.70   3.77   3.22   2.37   2.08   1.50   1.75   1.37      C_INV = 20
"""
import numpy as np
import pytest
import scipy.fft as sf
import scipy.signal

from oracle import ref_np as O
from test_chirpz_algorithm import czt_p, czt_sizes

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore")]

PAD_MODES = ("constant", "reflect", "edge", "symmetric", "linear_ramp")
INSTANCES = [1 << q for q in range(5, 13)]
U = 2.0 ** -24
C_FWD = 3.0                        # norm-wise bounds in units of u log2(P), see the module docstring
C_INV = 20.0


@pytest.fixture(scope="module")
def lb():
    import librosa_b200

    librosa_b200.default_context()
    return librosa_b200


def pairs_per_step(P):
    """G of the engine configuration: frame pairs per CTA step."""
    tpf = P // 32
    nw = 16 if P >= 1024 else tpf
    return nw * 32 // tpf


def sweep_sizes():
    """Every chirp-z frame length up to 256 (all of P = 32 ... 512); for P = 1024, 2048 and 4096 the first and last
    odd and even ones plus a seeded sample of eight more."""
    sizes = czt_sizes()
    out = [L for L in sizes if L <= 256]
    rng = np.random.default_rng(2047)
    for P in (1024, 2048, 4096):
        served = [L for L in sizes if czt_p(L) == P]
        odd, even = [L for L in served if L % 2], [L for L in served if L % 2 == 0]
        ends = {odd[0], odd[-1], even[0], even[-1]}
        rest = [L for L in served if L not in ends]
        out += sorted(ends | {int(L) for L in rng.choice(rest, 8, replace=False)})
    return out


def geometry(L, i):
    """stft keywords for the i-th size of a sweep: centre on and off, all pad modes, hops that do not divide n_fft,
    hop > n_fft, win_length < n_fft — spread over the sweep."""
    hop = [max(1, L // 4), L // 3 + 1, L // 2 + 1, max(1, 2 * L // 5 - 1)][i % 4]
    if i % 13 == 6:
        hop = L + L // 3 + 1
    win_length = max(2, L - L // 5 - 1) if i % 6 == 1 else None
    return dict(n_fft=L, hop_length=hop, win_length=win_length, center=i % 7 != 3, pad_mode=PAD_MODES[i % 5])


def burst(n_clips, n, L, seed):
    """-60 dB noise with one unit-level burst per clip (about half a frame to 1.5 frames long): paired frames differ
    in level by up to 60 dB."""
    rng = np.random.default_rng(seed)
    y = 1e-3 * rng.standard_normal((n_clips, n))
    for c in range(n_clips):
        s = int(rng.integers(0, n - 1))
        m = min(n - s, max(2, L // 2 + int(rng.integers(0, L + 1))))
        y[c, s:s + m] += 0.5 * rng.standard_normal(m) + 0.3 * np.sin(0.37 * np.arange(m))
    return y.astype(np.float32)


def window(L, win_length=None):
    return O.pad_center(scipy.signal.get_window("hann", win_length or L, fftbins=True), L)


def ref_stft(y, n_fft, hop_length, win_length=None, center=True, pad_mode="constant"):
    """float64 STFT, [..., frame, bin]."""
    y = np.asarray(y, dtype=np.float64)
    if center:
        y = np.pad(y, [(0, 0)] * (y.ndim - 1) + [(n_fft // 2, n_fft // 2)], mode=pad_mode)
    frames = np.lib.stride_tricks.sliding_window_view(y, n_fft, axis=-1)[..., ::hop_length, :]
    return sf.rfft(frames * window(n_fft, win_length), axis=-1)


def gpu_stft(lb, y, **kw):
    """stft of a float32 device batch, [..., frame, bin] complex64."""
    D = lb.stft(lb.to_device(y), **kw)
    assert isinstance(D, lb.DeviceArray) and D.dtype == np.complex64 and D.layout == "ft"
    return np.swapaxes(D.get(), -1, -2)


def to_device_ft(lb, D):
    """A [..., frame, bin] complex64 host spectrum as a device stft_matrix in the native layout."""
    D = np.ascontiguousarray(D, dtype=np.complex64)
    shape = D.shape[:-2] + (D.shape[-1], D.shape[-2])
    return lb.DeviceArray.empty(lb.default_context(), shape, np.complex64, layout="ft").set(D)


def gpu_istft(lb, D, **kw):
    y = lb.istft(to_device_ft(lb, D), **kw)
    assert isinstance(y, lb.DeviceArray) and y.dtype == np.float32
    return y.get()


def contract_close(got, ref, what, rtol=1e-4, atol_rel=1e-5):
    """|got - ref| <= rtol |ref| + atol_rel max|ref of the clip|, clip by clip (leading index)."""
    got = np.asarray(got)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    g = got.reshape(ref.shape[0], -1).astype(np.complex128 if np.iscomplexobj(got) else np.float64)
    r = ref.reshape(g.shape)
    for c in range(g.shape[0]):
        scale = float(np.abs(r[c]).max())
        err = np.abs(g[c] - r[c])
        bad = ~(err <= rtol * np.abs(r[c]) + atol_rel * scale)
        assert not bad.any(), f"{what} clip {c}: {int(bad.sum())} elements, max |err| / max|ref| = " \
                              f"{float(err.max()) / max(scale, 1e-300):.3e}"


def pair_ratio(got, ref):
    """max over frame pairs (2j, 2j+1 of a clip) of ||got - ref||_2 / (u max(||ref_A||, ||ref_B||)); got / ref are
    [clip, frame, sample-or-bin]."""
    e2 = (np.abs(got.astype(ref.dtype) - ref) ** 2).sum(axis=-1)
    n = np.sqrt((np.abs(ref) ** 2).sum(axis=-1))
    if e2.shape[-1] % 2:
        e2 = np.concatenate([e2, np.zeros_like(e2[..., :1])], axis=-1)
        n = np.concatenate([n, np.zeros_like(n[..., :1])], axis=-1)
    e = np.sqrt(e2[..., 0::2] + e2[..., 1::2])
    s = np.maximum(n[..., 0::2], n[..., 1::2])
    assert not e[s == 0].any()
    return float((e[s > 0] / s[s > 0]).max()) / U if (s > 0).any() else 0.0


def check_norm(ratio, P, what, inverse=False):
    C = C_INV if inverse else C_FWD
    assert ratio <= C * np.log2(P), f"{what}: ||err|| = {ratio / np.log2(P):.3f} u log2(P) max(||A||, ||B||) (bound {C})"


def istft_used_frames(T, n_fft, hop, center, length):
    if not length:
        return T
    return min(T, int(np.ceil((length + (2 * (n_fft // 2) if center else 0)) / hop)))


def ola_weights(n_fft, hop, win_length, n_frames, center, out_len):
    """The window-sum-square istft divides by, trimmed like istft (1 where it is tiny)."""
    wss = O.window_sumsquare("hann", n_frames, hop_length=hop, win_length=win_length, n_fft=n_fft, dtype=np.float64)
    wss = O.fix_length(wss[(n_fft // 2 if center else 0):], out_len)
    return np.where(wss > O.tiny(wss), wss, 1.0)


def istft_close(got, Din, kw, what):
    """istft of the complex64 spectrum Din ([clip, frame, bin]) against oracle.istft of the same values in float64,
    on the un-normalised overlap-add."""
    ref = O.istft(np.swapaxes(Din, -1, -2).astype(np.complex128), **kw)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    hop = kw["hop_length"]
    w = ola_weights(kw["n_fft"], hop, kw.get("win_length"),
                    istft_used_frames(Din.shape[-2], kw["n_fft"], hop, kw.get("center", True), kw.get("length")),
                    kw.get("center", True), ref.shape[-1])
    contract_close(got * w, ref * w, what)


def inverse_pair_ratio(lb, Din, L, win_length):
    """istft with hop = n_fft and no centring: output sample t belongs to frame t // n_fft alone, so y * wss is the
    window-weighted irfft of that frame — per-pair errors of czt_inv_kernel are observable."""
    y = gpu_istft(lb, Din, n_fft=L, hop_length=L, win_length=win_length, center=False)
    w = window(L, win_length)
    got = y.reshape(Din.shape[:-1] + (L,)).astype(np.float64) * w ** 2
    ref = sf.irfft(Din.astype(np.complex128), n=L, axis=-1) * w
    return pair_ratio(got, ref)


# ------------------------------------------------------------------ size sweep, forward and inverse
def sweep_case(lb, L, i):
    """Forward and inverse at frame length L with the i-th sweep geometry; returns the norm-wise ratios (in units of
    u, not yet divided by log2 P) of the forward and of the inverse."""
    kw = geometry(L, i)
    hop = kw["hop_length"]
    n = 3 * L + 7 * (i % 5) + 2 + (hop if hop > L else 0)
    y = burst(2, n, L, seed=L)
    ref = ref_stft(y, **kw)
    got = gpu_stft(lb, y, **kw)
    contract_close(got, ref, f"stft n_fft={L} {kw}")
    fwd = pair_ratio(got, ref)

    Din = ref.astype(np.complex64)
    # the output covers every sample the frames came from (a centred istft of natural length drops the signal's tail)
    length = None if not kw["center"] else (n if i % 2 else n + L // 3 + 1)
    ikw = dict(n_fft=L, hop_length=hop, win_length=kw["win_length"], center=kw["center"], length=length)
    istft_close(gpu_istft(lb, Din, **ikw), Din, ikw, f"istft n_fft={L} {ikw}")
    inv = inverse_pair_ratio(lb, Din, L, kw["win_length"])
    return fwd, inv


@pytest.mark.parametrize("P", INSTANCES)
def test_size_sweep_forward_and_inverse(lb, P):
    sweep = sweep_sizes()
    for i, L in enumerate(sweep):
        if czt_p(L) != P:
            continue
        fwd, inv = sweep_case(lb, L, i)
        check_norm(fwd, P, f"stft n_fft={L}")
        check_norm(inv, P, f"istft n_fft={L}", inverse=True)


# ------------------------------------------------------------------ |X|^power
# one odd frame length per instance, and one of either parity for the pairing tests
POWER_SIZES = {32: 15, 64: 27, 128: 51, 256: 99, 512: 201, 1024: 441, 2048: 1001, 4096: 1537}
PAIR_SIZES = {32: 14, 64: 28, 128: 49, 256: 98, 512: 255, 1024: 258, 2048: 1023, 4096: 1030}


def test_size_tables_are_chirpz_sizes():
    sizes = set(czt_sizes())
    for table in (POWER_SIZES, PAIR_SIZES):
        assert all(L in sizes and czt_p(L) == P for P, L in table.items())


@pytest.mark.parametrize("P", INSTANCES)
def test_power_modes(lb, P):
    """power 1 (sqrt.approx.f32 of |X|^2), 2 and 1.5 (power_from_sq) against |X_ref|^power."""
    L = POWER_SIZES[P]
    kw = dict(n_fft=L, hop_length=L // 3 + 1)
    y = burst(3, 5 * L + 3, L, seed=P)
    ref = np.abs(ref_stft(y, **kw))
    for power in (2.0, 1.0, 1.5):
        S, n_out = lb._spectrogram(y=lb.to_device(y), power=power, **kw)
        assert n_out == L and isinstance(S, lb.DeviceArray) and S.dtype == np.float32
        contract_close(np.swapaxes(S.get(), -1, -2), ref ** power, f"|X|^{power} n_fft={L}")


# ------------------------------------------------------------------ pairing and scheduling
@pytest.mark.parametrize("P", INSTANCES)
def test_frame_pairing_and_grid_stride(lb, P):
    """1, 2 and 3 frames per clip (the odd last frame rides alone with a zero partner); a pair count that is not a
    multiple of G (spare groups redo the last pair with their stores masked); a batch of more than 3 sm_count G pairs
    (the grid holds one block per SM, so the grid-stride loop runs several times).  Every clip of a batch equals the
    clip computed alone, bit for bit."""
    L = PAIR_SIZES[P]
    G = pairs_per_step(P)
    ctx = lb.default_context()
    hop = L // 2 + 1
    big = (3 * ctx.sm_count * G) // 5 + 7
    batches = [(5, 1), (5, 2), (5, 3),                                     # frames per clip
               (G // 2 + 3, 3),                                            # G + 6 pairs
               (big, 9)]                                                   # 5 big > 3 sm_count G pairs
    assert (G + 6) % G and 5 * big > 3 * ctx.sm_count * G
    for n_clips, T in batches:
        n = L + hop * (T - 1)
        kw = dict(n_fft=L, hop_length=hop, center=False)
        y = burst(n_clips, n, L, seed=P + n_clips + T)
        ref = ref_stft(y, **kw)
        got = gpu_stft(lb, y, **kw)
        assert got.shape == ref.shape and got.shape[-2] == T
        contract_close(got, ref, f"stft n_fft={L} clips={n_clips} T={T}")
        check_norm(pair_ratio(got, ref), P, f"stft n_fft={L} clips={n_clips} T={T}")
        for c in sorted({0, 1, n_clips // 2, n_clips - 2, n_clips - 1}):
            np.testing.assert_array_equal(got[c], gpu_stft(lb, y[c:c + 1], **kw)[0], err_msg=f"clip {c} of {n_clips}")
        Din = ref.astype(np.complex64)
        ikw = dict(n_fft=L, hop_length=hop, center=False)
        yr = gpu_istft(lb, Din, **ikw)
        istft_close(yr, Din, ikw, f"istft n_fft={L} clips={n_clips} T={T}")
        for c in sorted({0, n_clips - 1}):
            np.testing.assert_array_equal(yr[c], gpu_istft(lb, Din[c:c + 1], **ikw)[0])
        check_norm(inverse_pair_ratio(lb, Din, L, None), P, f"istft n_fft={L} clips={n_clips} T={T}", inverse=True)


@pytest.mark.parametrize("P", INSTANCES)
def test_clips_are_isolated(lb, P):
    """Pairs never straddle clips: a clip 80 dB louder next to a quiet one leaves the quiet clip at its own relative
    accuracy, forward and inverse, and a NaN clip poisons only itself."""
    L = POWER_SIZES[P]
    kw = dict(n_fft=L, hop_length=L // 3 + 1)
    n = 4 * L + 1
    y = burst(4, n, L, seed=3 * P).astype(np.float64)
    y[0::2] *= 1e4
    T = 1 + (n + 2 * (L // 2) - L) // kw["hop_length"]
    if T % 2 == 0:                                                         # odd frame count: a lone last frame
        n += kw["hop_length"]
        y = np.concatenate([y, y[:, :kw["hop_length"]]], axis=1)
    y = y.astype(np.float32)
    ref = ref_stft(y, **kw)
    assert ref.shape[-2] % 2 == 1
    got = gpu_stft(lb, y, **kw)
    contract_close(got, ref, f"stft n_fft={L} loud/quiet")                # relative to each clip's own peak
    Din = ref.astype(np.complex64)
    ikw = dict(n_fft=L, hop_length=kw["hop_length"], length=n)
    istft_close(gpu_istft(lb, Din, **ikw), Din, ikw, f"istft n_fft={L} loud/quiet")
    yn = y.copy()
    yn[2, n // 2] = np.nan
    bad = gpu_stft(lb, yn, **kw)
    assert np.isnan(bad[2]).any()
    for c in (0, 1, 3):
        np.testing.assert_array_equal(bad[c], got[c])


# ------------------------------------------------------------------ irfft semantics of every inverse family
def irfft_sizes():
    sizes = czt_sizes()
    out = []
    for P in INSTANCES:
        served = [L for L in sizes if czt_p(L) == P]
        out += [next(L for L in served[len(served) // 2:] if L % 2), next(L for L in served[len(served) // 2:] if L % 2 == 0)]
    return out


@pytest.mark.parametrize("family,sizes", [("chirpz", None), ("mixed_radix", [12, 400, 4000]),
                                          ("pow2", [8, 128, 2048, 8192])])
def test_istft_ignores_imaginary_dc_and_nyquist(lb, family, sizes):
    """scipy.fft.irfft ignores Im of the DC bin, and of the Nyquist bin for even n_fft; so must czt_inv_kernel,
    mr_inv_kernel and inv_kernel.  The spectra here carry random imaginary parts there as large as the largest bin."""
    rng = np.random.default_rng(11)
    for L in sizes or irfft_sizes():
        hop = max(1, L // 4)
        n = 4 * L + 5
        y = burst(2, n, L, seed=L + 1)
        Din = ref_stft(y, n_fft=L, hop_length=hop)
        scale = float(np.abs(Din).max())
        Din[..., 0] += 1j * scale * rng.uniform(0.5, 1.0, Din.shape[:-1]) * rng.choice([-1, 1], Din.shape[:-1])
        if L % 2 == 0:
            Din[..., -1] += 1j * scale * rng.uniform(0.5, 1.0, Din.shape[:-1]) * rng.choice([-1, 1], Din.shape[:-1])
        Din = Din.astype(np.complex64)
        ikw = dict(n_fft=L, hop_length=hop, length=n)
        istft_close(gpu_istft(lb, Din, **ikw), Din, ikw, f"{family} istft n_fft={L}")


# ------------------------------------------------------------------ composed consumers
COMPOSED_SIZES = [13, 23, 45, 101, 243, 501, 999, 1537]


@pytest.mark.parametrize("L", COMPOSED_SIZES)
def test_composed_consumers(lb, L):
    """melspectrogram / mfcc / spectral_centroid / chroma_stft from y, and griffinlim, at one size per instance, on
    the tolerances of test_gpu_parity / test_gpu_features."""
    import signals

    assert sorted({czt_p(x) for x in COMPOSED_SIZES}) == INSTANCES
    y = signals.make("B", (2, 6 * L + 1000), seed=L)
    hop = L // 4 + 1
    n_mels = min(40, max(4, L // 8))
    kw = dict(sr=22050, n_fft=L, hop_length=hop)
    d = lb.to_device(y)

    def got(x):
        return x.get() if isinstance(x, lb.DeviceArray) else x

    ref = O.melspectrogram(y=y, n_mels=n_mels, **kw)
    contract_close(got(lb.feature.melspectrogram(y=d, n_mels=n_mels, **kw)), ref, f"mel n_fft={L}", atol_rel=1e-6)
    n_mfcc = min(13, n_mels)
    ref = O.mfcc(y=y, n_mfcc=n_mfcc, n_mels=n_mels, **kw)
    np.testing.assert_allclose(got(lb.feature.mfcc(y=d, n_mfcc=n_mfcc, n_mels=n_mels, **kw)), ref, rtol=1e-4, atol=1e-3)
    ref = O.spectral_centroid(y=y, **kw)
    contract_close(got(lb.feature.spectral_centroid(y=d, **kw)), ref, f"centroid n_fft={L}", atol_rel=1e-6)
    ref = O.chroma_stft(y=y, tuning=0.0, **kw)
    np.testing.assert_allclose(got(lb.feature.chroma_stft(y=d, tuning=0.0, **kw)), ref, rtol=1e-4, atol=2e-6)
    S = np.abs(O.stft(y[0], n_fft=L, hop_length=hop))
    g = lb.griffinlim(S, n_iter=1, rng=0, n_fft=L, hop_length=hop)
    want = O.griffinlim(S, n_iter=1, rng=0, n_fft=L, hop_length=hop)
    assert g.shape == want.shape and g.dtype == want.dtype
    np.testing.assert_allclose(g, want, rtol=0, atol=2e-3 * float(np.abs(want).max()))


# ------------------------------------------------------------------ util.valid_audio at chirp-z sizes
@pytest.mark.parametrize("L", [21, 501])
def test_nonfinite_input_raises_like_valid_audio(lb, L):
    """A NaN / +-inf inside a frame, in a hop gap and in the tail no frame reads: ParameterError through stft,
    melspectrogram and mfcc; the next clean call passes (the status flag does not stick)."""
    n = 40 * L + 3
    y = burst(2, n, L, seed=L)
    gap_hop = L + L // 2 + 1
    tail_hop = L // 2 + 2
    tail_T = 1 + (n - L) // tail_hop
    assert (tail_T - 1) * tail_hop + L < n
    positions = [(n // 2, dict(hop_length=L // 4 + 1)),
                 (L + 1, dict(hop_length=gap_hop, center=False)),
                 (n - 1, dict(hop_length=tail_hop, center=False))]
    fns = (lambda a, kw: lb.stft(a, n_fft=L, **kw),
           lambda a, kw: lb.feature.melspectrogram(y=a, n_fft=L, n_mels=8, **kw),
           lambda a, kw: lb.feature.mfcc(y=a, n_fft=L, n_mels=8, n_mfcc=8, **kw))
    for pos, kw in positions:
        for bad in (np.nan, np.inf, -np.inf):
            z = y.copy()
            z[1, pos] = bad
            for fn in fns:
                with pytest.raises(lb.ParameterError, match="not finite everywhere"):
                    fn(z, kw)
            for fn in fns:
                assert np.isfinite(fn(y, kw)).all()


# ------------------------------------------------------------------ route
def test_every_swept_size_takes_the_chirpz_route(lb):
    """Same launches per stft / istft / melspectrogram call as n_fft = 501 (one chirp-z kernel, plus the overlap-add
    of the inverse and the mel projection), for every size of the sweep."""
    ctx = lb.default_context()

    def counts(L):
        hop = L // 4 + 1
        y = lb.to_device(burst(2, 4 * L, L, seed=1))
        D = lb.stft(y, n_fft=L, hop_length=hop)
        out = []
        for call in (lambda: lb.stft(y, n_fft=L, hop_length=hop),
                     lambda: lb.istft(D, n_fft=L, hop_length=hop),
                     lambda: lb.feature.melspectrogram(y=y, n_fft=L, hop_length=hop, n_mels=8)):
            before = ctx.launch_count
            call()
            out.append(ctx.launch_count - before)
        return out

    want = counts(501)
    assert want[0] == 1
    got = {L: counts(L) for L in sweep_sizes()}
    assert {L: c for L, c in got.items() if c != want} == {}

