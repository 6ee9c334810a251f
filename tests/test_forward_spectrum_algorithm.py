"""The host side of the STFT, spectrogram and spectral-statistics paths restated in integer-indexed NumPy, on the CPU:
which fwd_kernel instance serves MODE_STFT / MODE_SPEC / MODE_STATS, how stats_kernel is sized, how frame_stats splits
a row over the lanes of a warp, and how many warps mr_kernel runs in modes 0 and 1.  This file is the specification
the kernels are read against; tests/test_gpu_forward_spectrum.py runs them.

Restated here:
    run_forward                      forward_choice of tests/test_mel_front_end_algorithm.py with its `mode`: no
      (csrc/spectrum_api.cu)         MelRow table outside MODE_MEL, the M + 1 bin frequencies in MODE_STATS, and an
                                     exchange region of FT (M + M/32) float2 in MODE_STFT / MODE_SPEC against the
                                     MelLayout group stride in MODE_STATS
    b2l_spectral_stats_from_spec     stats_kernel's warp ladder nw = 8 -> 4 -> 2 -> 1: the first nw whose block,
      (csrc/feature_api.cu)          (nw + 1) Fp 4 bytes with Fp = (F + 3) & ~3, fits the opt-in shared memory
    frame_stats (csrc/stats.cuh)     lane l owns bins [l c, (l + 1) c) clipped to F, c = ((F + 31) / 32) | 1; the
                                     running sum of bin k is the exclusive warp scan of the chunk totals (shfl_up,
                                     Hillis-Steele) plus the lane-local walk
    mr_block                         warps per block of mr_kernel<0 | 1, G> (no mel tables), G = 16 lanes per frame for
      (csrc/spectrum_api.cu)         M <= 512, 32 above

The selection tables are H100 constants (232 448 bytes of opt-in shared memory).  Last, the comparisons the GPU test
uses must reject subtly wrong kernels simulated in float64 on that test's own signals.
"""
import numpy as np
import pytest

from test_inverse_gather_algorithm import H100_SMEM_OPTIN
from test_mel_front_end_algorithm import (MODE_MEL, MODE_SPEC, MODE_STATS, MODE_STFT, SIZES, forward_choice,
                                          mr_sizes, mr_table_bytes, mr_tw_count, variant_runs)

# MODE_STFT and MODE_SPEC (same shared-memory layout): (first hop, last hop, variant, FT) per size, then the first
# refused hop.  116 = two 8-warp halves.
H100_SPECTRUM_VARIANTS = {
    8: ([(1, 1865, 1, 32)], 1866),
    16: ([(1, 1856, 1, 32)], 1857),
    32: ([(1, 1838, 1, 32)], 1839),
    64: ([(1, 1801, 1, 32)], 1802),
    128: ([(1, 1726, 2, 32)], 1727),
    256: ([(1, 1578, 4, 32)], 1579),
    512: ([(1, 1281, 8, 32)], 1282),
    1024: ([(1, 674, 116, 16), (675, 686, 16, 32)], 687),
    2048: ([(1, 1248, 116, 8), (1249, 1303, 16, 16), (1304, 5206, 8, 8)], 5207),
    4096: ([(1, 1546, 116, 4), (1547, 1915, 16, 8), (1916, 10101, 8, 4)], 10102),
    8192: ([(1, 16672, 8, 2)], 16673),
}

# MODE_STATS: the same instances, narrower windows (frequency table, MelLayout exchange stride).
H100_STATS_VARIANTS = {
    8: ([(1, 1835, 1, 32)], 1836),
    16: ([(1, 1834, 1, 32)], 1835),
    32: ([(1, 1833, 1, 32)], 1834),
    64: ([(1, 1796, 1, 32)], 1797),
    128: ([(1, 1721, 2, 32)], 1722),
    256: ([(1, 1545, 4, 32)], 1546),
    512: ([(1, 1252, 8, 32)], 1253),
    1024: ([(1, 652, 116, 16), (653, 665, 16, 32)], 666),
    2048: ([(1, 1165, 116, 8), (1166, 1230, 16, 16), (1231, 5051, 8, 8)], 5052),
    4096: ([(1, 1194, 116, 4), (1195, 1613, 16, 8), (1614, 9408, 8, 4)], 9409),
    8192: ([(1, 12544, 8, 2)], 12545),
}

# stats_kernel: (warps per block, largest n_bins served with them); n_bins 29 057 and up are refused.
STATS_LADDER = [(8, 6456), (4, 11620), (2, 19368), (1, 29056)]

# mr_kernel<0 | 1, G>: (first n_fft, last n_fft, warps per block) over the 96 mixed-radix sizes in increasing order.
H100_MR_SPECTRUM_WARPS = [
    (12, 432, 16), (450, 450, 15), (480, 486, 14), (500, 500, 13), (540, 540, 12), (576, 600, 11), (640, 648, 10),
    (720, 750, 9), (768, 810, 8), (864, 900, 7), (960, 1000, 6), (1080, 1080, 12), (1152, 1152, 11),
    (1200, 1280, 10), (1296, 1350, 9), (1440, 1536, 8), (1600, 1728, 7), (1800, 1944, 6), (2000, 2304, 5),
    (2400, 2700, 4), (2880, 3240, 3), (3456, 4050, 2),
]


# ------------------------------------------------------------------ b2l_spectral_stats_from_spec (feature_api.cu)
def stats_block(F, smem_optin=H100_SMEM_OPTIN):
    """(warps per block, shared-memory bytes) of stats_kernel for rows of F bins, or None (refused)."""
    Fp = (F + 3) & ~3
    nw = 8
    while nw > 1 and (nw + 1) * Fp * 4 > smem_optin:
        nw >>= 1
    smem = (nw + 1) * Fp * 4
    return None if smem > smem_optin else (nw, smem)


# ------------------------------------------------------------------ frame_stats (stats.cuh)
def chunk_of(F):
    """Bins per lane: odd, so that the warp-wide access row[l c + i] touches 32 distinct banks."""
    return ((F + 31) // 32) | 1


def lane_ranges(F):
    """[k0, k1) of lanes 0 .. 31 for rows of F bins (arrays broadcast over F)."""
    F = np.asarray(F)[..., None]
    c = chunk_of(F)
    lane = np.arange(32)
    k0 = np.minimum(F, lane * c)
    k1 = np.minimum(F, k0 + c)
    return k0, k1


def warp_exclusive_scan(x):
    """The shfl_up Hillis-Steele scan of frame_stats over the last axis (32 lanes), minus the own term."""
    incl = x.copy()
    o = 1
    while o < 32:
        up = np.zeros_like(incl)
        up[..., o:] = incl[..., :-o]                                     # shfl_up: lanes < o keep their own value
        incl = incl + up                                                 # (and do not add it)
        o <<= 1
    return incl - x, incl[..., 31]


# ------------------------------------------------------------------ mr_block (spectrum_api.cu), modes 0 and 1
def mr_spectrum_block(n_fft, smem_optin=H100_SMEM_OPTIN):
    """(lanes per frame G, warps per block, shared-memory bytes) of run_mr in modes 0 / 1 (n_mels 0), or None."""
    M = n_fft // 2
    fpw = 2 if M <= 512 else 1
    tables = mr_table_bytes(n_fft, mr_tw_count(n_fft), 0, 0)
    per_warp = 2 * M * 8 * fpw
    budget = (smem_optin + 1024) // 2 - 1024
    w = 16
    while w > 1 and tables + w * per_warp > budget:
        w -= 1
    if tables + w * per_warp > smem_optin:
        return None
    return 32 // fpw, w, tables + w * per_warp


# ================================================================== tests
@pytest.mark.parametrize("n_fft", SIZES)
def test_spectrum_selection_table(n_fft):
    """MODE_STFT and MODE_SPEC select the same instance at every hop up to the first refused one."""
    got = variant_runs(n_fft, None, mode=MODE_STFT)
    assert got == H100_SPECTRUM_VARIANTS[n_fft]
    assert variant_runs(n_fft, None, mode=MODE_SPEC) == got
    for first, last, v, f in got[0]:
        c = forward_choice(n_fft, last, None, mode=MODE_STFT)
        M = n_fft // 2
        assert c[:3] == (v, f, 2 if v == 116 else 1) and c[3] <= H100_SMEM_OPTIN
        assert c[4] == -(-f * (M + M // 32) * 8 // 128) * 128              # the plain exchange region


@pytest.mark.parametrize("n_fft", SIZES)
def test_stats_selection_table(n_fft):
    """MODE_STATS: the same instances as the spectrum modes, each window ending no later (the frequency table and
    the MelLayout group stride only add shared memory), and a MODE_MEL basis plays no part."""
    got = variant_runs(n_fft, None, mode=MODE_STATS)
    assert got == H100_STATS_VARIANTS[n_fft]
    spec = H100_SPECTRUM_VARIANTS[n_fft]
    assert [r[2:] for r in got[0]] == [r[2:] for r in spec[0]]
    assert all(a[1] <= b[1] for a, b in zip(got[0], spec[0])) and got[1] <= spec[1]


def test_modes_differ_from_the_mel_windows():
    """The mel test's instance table does not carry over: the windows of every mode differ at n_fft 1024 ... 4096."""
    from test_mel_front_end_algorithm import H100_MEL_VARIANTS

    for n_fft in (1024, 2048, 4096):
        assert H100_MEL_VARIANTS[n_fft] != H100_SPECTRUM_VARIANTS[n_fft] != H100_STATS_VARIANTS[n_fft]
    assert MODE_MEL not in (MODE_STFT, MODE_SPEC, MODE_STATS)


def test_stats_kernel_ladder():
    """Warps per block as a function of n_bins: 8 up to 6 456 bins, 4 up to 11 620, 2 up to 19 368, 1 up to 29 056,
    refused above; each block fits the opt-in shared memory."""
    prev = 1
    for nw, last in STATS_LADDER:
        assert stats_block(prev + 1)[0] == nw and stats_block(last)[0] == nw
        assert stats_block(last)[1] <= H100_SMEM_OPTIN
        prev = last
    assert stats_block(2)[0] == 8 and stats_block(STATS_LADDER[-1][1] + 1) is None
    F = np.arange(2, 29060)
    nws = np.array([b[0] if b else 0 for b in map(stats_block, F)])
    assert (np.diff(nws) <= 0).all()                                     # one rung after the other


def test_frame_stats_partition():
    """For every F from 2 to 29 056: the lane chunks cover [0, F) exactly once, in lane order, and lanes at or past
    the end get empty ranges."""
    F = np.arange(2, STATS_LADDER[-1][1] + 1)
    k0, k1 = lane_ranges(F)
    c = chunk_of(F)[:, None]
    assert (c % 2 == 1).all() and (32 * c >= F[:, None]).all()
    assert (k0[:, 0] == 0).all() and (k1[:, -1] == F).all()
    assert (k1[:, :-1] == k0[:, 1:]).all()                               # contiguous, no gap, no overlap
    assert ((k1 - k0).sum(axis=1) == F).all()
    past = np.arange(32)[None, :] * c >= F[:, None]
    assert (k0[past] == k1[past]).all() and (k1[past] == np.broadcast_to(F[:, None], past.shape)[past]).all()
    assert past.any()                                                    # some F leave lanes idle (e.g. F = 33)


def test_frame_stats_scan_reproduces_cumsum():
    """On integer data the exclusive warp scan of the chunk totals plus the lane-local walk is cumsum exactly: for
    every F from 2 to 29 056 at the chunk boundaries, and bin by bin for F up to 2 048 and the ladder ends."""
    rng = np.random.default_rng(0)
    top = STATS_LADDER[-1][1]
    data = rng.integers(0, 1 << 20, size=top + 1).astype(np.int64)
    P = np.concatenate([[0], np.cumsum(data)])
    F = np.arange(2, top + 1)
    k0, k1 = lane_ranges(F)
    excl, total = warp_exclusive_scan(P[k1] - P[k0])
    assert (excl == P[k0]).all() and (total == P[F]).all()
    for f in list(range(2, 2049)) + [b for _, b in STATS_LADDER] + [b + 1 for _, b in STATS_LADDER[:-1]]:
        a0, a1 = lane_ranges(f)
        row = data[:f]
        ex, _ = warp_exclusive_scan(np.array([row[a0[lane]:a1[lane]].sum() for lane in range(32)]))
        run = np.empty(f, np.int64)
        for lane in range(32):
            run[a0[lane]:a1[lane]] = ex[lane] + np.cumsum(row[a0[lane]:a1[lane]])
        assert (run == np.cumsum(row)).all(), f


def test_mixed_radix_spectrum_blocks():
    """mr_kernel<0 | 1, G> at all 96 mixed-radix sizes: G = 16 lanes per frame up to n_fft 1024 (M <= 512), 32
    above; the pinned warps per block; two blocks per SM."""
    sizes = mr_sizes()
    assert len(sizes) == 96
    want = {}
    for first, last, w in H100_MR_SPECTRUM_WARPS:
        for n in sizes:
            if first <= n <= last:
                want[n] = w
    assert sorted(want) == sizes
    for n_fft in sizes:
        G, w, smem = mr_spectrum_block(n_fft)
        assert G == (16 if n_fft // 2 <= 512 else 32) and w == want[n_fft], n_fft
        assert smem <= (H100_SMEM_OPTIN + 1024) // 2 - 1024


# ------------------------------------------------------------------ sensitivity of the GPU test's comparisons
def round_mantissa(x, bits):
    m, e = np.frexp(x)
    return np.ldexp(np.round(m * 2.0 ** bits) / 2.0 ** bits, e)


def rfft_rounded_twiddles(frames, bits):
    """rfft in float64 by a four-step transform (N = N1 N2) whose inter-pass twiddles W_N^(n2 k1) are rounded to
    `bits` mantissa bits: what a split twiddle table rounded that far computes."""
    N = frames.shape[-1]
    N1 = 1 << (int(np.log2(N)) // 2)
    N2 = N // N1
    x = frames.reshape(frames.shape[:-1] + (N1, N2))                     # x[N2 n1 + n2]
    A = np.fft.fft(x, axis=-2)                                           # [k1, n2]
    ang = -2.0 * np.pi * np.outer(np.arange(N1), np.arange(N2)) / N
    tw = round_mantissa(np.cos(ang), bits) + 1j * round_mantissa(np.sin(ang), bits)
    B = np.fft.fft(A * tw, axis=-1)                                      # [k1, k2]
    X = np.swapaxes(B, -1, -2).reshape(frames.shape[:-1] + (N,))         # X[k1 + N1 k2]
    return X[..., :N // 2 + 1]


def inclusive_rolloff(S, freq, roll):
    """The roll-off a frame_stats whose scan is inclusive would report: every running sum one chunk total ahead."""
    F = S.shape[-1]
    k0, k1 = lane_ranges(F)
    lane = np.searchsorted(k1, np.arange(F), side="right")
    P = np.concatenate([np.zeros(S.shape[:-1] + (1,)), np.cumsum(S, axis=-1)], axis=-1)
    own = (P[..., k1] - P[..., k0])[..., lane]
    wrong = np.cumsum(S, axis=-1) + own
    f = freq.astype(np.float64)
    return np.where(wrong >= roll * S.sum(axis=-1)[..., None], f, np.inf).min(axis=-1).astype(np.float32)


@pytest.mark.parametrize("n_fft", [8, 64, 512, 2048, 8192])
def test_comparison_rejects_subtly_wrong_kernels(n_fft):
    """The GPU test's comparisons, fed float32-rounded float64 results of wrong kernels on its own signals: the
    right result passes; the split twiddle table rounded to 12 mantissa bits (by the norm-wise bound), the middle
    bin conjugated, and the roll-off of an inclusive scan (fused and stats_kernel checks) are rejected."""
    import scipy.fft as sf

    import test_gpu_forward_spectrum as G
    from test_gpu_chirpz import window

    hop = n_fft // 4
    ft = forward_choice(n_fft, hop, None, mode=MODE_STFT)[1]
    y = G.signals(3, G.n_samples(2 * ft + 1, n_fft, hop, True), n_fft, seed=n_fft)
    X64 = G.ref_spectrum(y, n_fft, hop)
    G.stft_close(X64.astype(np.complex64), X64, n_fft, "exact")
    # split twiddle table rounded to 12 mantissa bits
    yp = np.pad(y.astype(np.float64), [(0, 0), (n_fft // 2, n_fft // 2)])
    frames = np.lib.stride_tricks.sliding_window_view(yp, n_fft, axis=-1)[:, ::hop] * window(n_fft)
    np.testing.assert_allclose(rfft_rounded_twiddles(frames, 52), sf.rfft(frames, axis=-1), rtol=0, atol=1e-12)
    wrong = rfft_rounded_twiddles(frames, 12).astype(np.complex64)
    assert G.norm_ratio(wrong, X64) / np.log2(n_fft) > G.C_STFT          # the norm-wise bound alone rejects it
    with pytest.raises(AssertionError):
        G.stft_close(wrong, X64, n_fft, "12-bit twiddles")
    with pytest.raises(AssertionError):
        G.spec_close((np.abs(wrong) ** 2).astype(np.float32), X64, n_fft, 2.0, "12-bit twiddles")
    # middle bin conjugated
    mid = X64.copy()
    mid[..., n_fft // 4] = np.conj(mid[..., n_fft // 4])
    with pytest.raises(AssertionError):
        G.stft_close(mid.astype(np.complex64), X64, n_fft, "middle bin conjugated")
    # roll-off from an inclusive scan: the fused check and the stats_kernel check
    freq = G.fft_freq(22050, n_fft)
    S64 = np.abs(X64)
    rows = G.ref_stats(S64, freq.astype(np.float64), frame_length=n_fft).astype(np.float32)
    G.fused_stats_close(rows, X64, freq, n_fft, "exact", n_fft)
    bad = rows.copy()
    bad[:, 2] = inclusive_rolloff(S64, freq, np.float32(0.85))
    assert (bad[:, 2] != rows[:, 2]).any()
    with pytest.raises(AssertionError, match="roll-off"):
        G.fused_stats_close(bad, X64, freq, n_fft, "inclusive scan", n_fft)
    S32 = S64.astype(np.float32)
    rows32 = G.ref_stats(S32, freq, frame_length=n_fft).astype(np.float32)
    G.stats_exact_check(rows32, S32, freq, "exact", frame_length=n_fft)
    rows32[:, 2] = inclusive_rolloff(S32.astype(np.float64), freq, np.float32(0.85))
    with pytest.raises(AssertionError, match="roll-off"):
        G.stats_exact_check(rows32, S32, freq, "inclusive scan", frame_length=n_fft)
