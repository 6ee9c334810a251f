"""The host side of the fused mel / MFCC front end restated in integer-indexed NumPy, on the CPU: which kernel
instance serves a call, the MelRow table the power-of-two kernel projects with, and the DCT kernel that follows.
This file is the specification the kernels are read against; tests/test_gpu_mel_front_end.py runs them.

Restated here:
    build_mel (csrc/plan.cu)         band extents [lo, lo + len) of every row of the float32 basis
    get_row_table (csrc/plan.cu)     the MelRow table for H rows per warp: start bins lo (a multiple of 4, bank
                                     rule lo == 4 (j mod G) mod max(H, 4)), shared trip count `quads` per work item,
                                     zero-padded weights at `off`
    MelLayout (csrc/common.cuh)      rows per warp H, group stride GS, row stride RS = 2 GS
    run_forward                      MODE_MEL: CTA variant (116 = two 8-warp halves, then 16, then 8 warps), frames
      (csrc/spectrum_api.cu)         per tile FT, halves and the shared-memory bytes, the first that fits wins
    mr_block / run_mr                warps per block and lanes per frame G of mr_kernel
      (csrc/spectrum_api.cu)
    launch_dct                       dct_clamp4_kernel with KS = 2 or 1 warp sets, dct_generic_kernel, or refused
      (csrc/spectrum_api.cu)

Asserted over a grid of mel configurations crossed with every (n_fft, FT) an H100 reaches: every shared-memory word a
row reads is one the same tile wrote for the same frame (its power row, bins 0 .. M + 3, or a non-padding word of the
frame's exchange region), and the last frame of a tile stays inside the allocation; the padded weights are the basis
bit for bit with exact zeros around it; the padded-row projection equals basis @ P.  The selection tables are H100
constants (232 448 bytes of opt-in shared memory).  Last, the comparison the GPU test uses must reject three subtly
wrong kernels simulated in float64 on the GPU test's own signals.
"""
import itertools
import warnings

import numpy as np
import pytest

from librosa_b200 import filters
from test_inverse_gather_algorithm import H100_SMEM_OPTIN, align_up
from test_mixed_radix_algorithm import mr_factor

SIZES = [2 << q for q in range(2, 13)]     # n_fft 8 ... 8192 (fwd_inst.cu)
TW_SPLIT_ROWS = 10                         # kTwSplitRows (fft_engine.cuh): (8 - 1) + (32 / 8 - 1)
NORMS = [None, "slaney", 1, 2, np.inf]


def mel_basis(sr, n_fft, n_mels=128, fmin=0.0, fmax=None, htk=False, norm="slaney"):
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                                  # empty filters
        return filters.mel(sr=sr, n_fft=n_fft, n_mels=n_mels, fmin=fmin, fmax=fmax, htk=htk, norm=norm)


# ------------------------------------------------------------------ MelLayout (common.cuh)
def rows_per_warp(ft):
    """H: PAIR tiles (FT even, >= 8) give each lane two frames, FP = FT / 2 lanes along frames."""
    return 32 // (ft // 2 if ft % 2 == 0 and ft >= 8 else ft)


def group_stride(M, ft):
    rsm = max(rows_per_warp(ft), 4)
    xb = M + M // 32
    return xb + ((rsm - 2 * xb) % 32) // 2


def xphys(e):
    return e + (e >> 5)


def written_words(M):
    """Words of a frame's exchange region the tile writes before the mel phase reads it: the power row (bins
    0 .. M plus three zeros) and the float2 exchange slots the FFT stores — every slot for a multi-pass transform,
    the un-mix stores of the upper half (e >= M / 2) for the one-pass transforms of M <= 32."""
    tpf = M // 32 if M >= 32 else 1
    ppt = M // tpf
    one_pass = ppt == M
    e = np.arange(M // 2 if one_pass else 0, M)
    p = xphys(e)
    out = np.zeros(2 * (M + M // 32) + 64, dtype=bool)
    out[2 * p] = out[2 * p + 1] = True
    out[:M + 4] = True
    return out


# ------------------------------------------------------------------ build_mel / get_row_table (plan.cu)
def bands(basis):
    """(lo, len) of every row: first and last non-zero bin; (0, 0) for an empty row."""
    out = []
    for r in basis:
        nz = np.flatnonzero(r != 0)
        out.append((0, 0) if nz.size == 0 else (int(nz[0]), int(nz[-1] - nz[0] + 1)))
    return out


class RowTable:
    def __init__(self, lo, quads, off, w, n_rows):
        self.lo, self.quads, self.off, self.w, self.n_rows = lo, quads, off, w, n_rows


def row_table(basis, H):
    n_mels = basis.shape[0]
    bs = bands(basis)
    rsm = max(H, 4)
    G = rsm // 4
    n_rows = -(-n_mels // H) * H
    lo = np.zeros(n_rows, np.int64)
    quads = np.zeros(n_rows, np.int64)
    off = np.zeros(n_rows, np.int64)
    w = []
    for item in range(n_rows // H):
        start, lenp = [], []
        for j in range(H):
            m = item * H + j
            if m < n_mels and bs[m][1] > 0:
                b_lo, b_len = bs[m]
                want = 4 * (j % G)
                st = b_lo - ((b_lo - want) % rsm)
                if st < 0:
                    st = b_lo - b_lo % 4
                start.append(st)
                lenp.append(b_lo + b_len - st)
            else:
                start.append(4 * (j % G))
                lenp.append(0)
        q = max((x + 3) // 4 for x in lenp)
        for j in range(H):
            m = item * H + j
            lo[m], quads[m], off[m] = start[j], q, len(w)
            row = [0.0] * (4 * q)
            if lenp[j] > 0:
                b_lo, b_len = bs[m]
                row[b_lo - start[j]:b_lo - start[j] + b_len] = basis[m, b_lo:b_lo + b_len].tolist()
            w.extend(row)
    return RowTable(lo, quads, off, np.asarray(w, dtype=np.float32), n_rows)


def dense_rows(t, M, RS):
    """The padded rows scattered back to [n_rows][RS] words (float64): what lane j multiplies word k of a frame by."""
    out = np.zeros((t.n_rows, RS + 4 * int(t.quads.max(initial=0))))
    for m in range(t.n_rows):
        q = int(t.quads[m])
        out[m, t.lo[m]:t.lo[m] + 4 * q] = t.w[t.off[m]:t.off[m] + 4 * q]
    return out


# ------------------------------------------------------------------ run_forward (spectrum_api.cu), MODE_MEL
def tw_count_split(log2m):
    """HostFftCfg::tw_count(true): fwd_kernel's split inter-pass table."""
    M = 1 << log2m
    tpf = M // 32 if M >= 32 else 1
    ppt = M // tpf
    logp = int(np.log2(ppt))
    npass = 1 if ppt == 1 else (log2m + logp - 1) // logp
    count = 0
    for q in range(1, npass):
        radix = 1 << min(logp, log2m - q * logp)
        rows = TW_SPLIT_ROWS if radix == 32 and log2m <= 11 else radix - 1
        count += rows << (q * logp)
    return count


MODE_STFT, MODE_MEL, MODE_SPEC, MODE_STATS = 0, 1, 2, 3                   # FwdMode (common.cuh)


def forward_choice(n_fft, hop, basis, smem_optin=H100_SMEM_OPTIN, mode=MODE_MEL):
    """(variant, FT, halves, shared-memory bytes, per-half exchange bytes) of run_forward in `mode`, or None
    (refused).  The modes differ in the tables after the mbarriers (the MelRow table in MODE_MEL, the M + 1 bin
    frequencies in MODE_STATS, nothing in MODE_STFT / MODE_SPEC) and in the exchange region: the MelLayout group
    stride where the power rows are parked (MODE_MEL, MODE_STATS), the plain FT (M + M / 32) float2 otherwise.
    `basis` is only read in MODE_MEL."""
    log2m = int(np.log2(n_fft)) - 1
    M, N = n_fft // 2, n_fft
    tpf = M // 32 if M >= 32 else 1
    variants = ([116] if 9 <= log2m <= 11 else []) + ([16, 8] if log2m >= 10 else [min(16, tpf)])
    for v in variants:
        nw, nh = (16, 2) if v == 116 else (v, 1)
        if nw * 32 % (tpf * nh):
            continue
        f = nw * 32 // nh // tpf
        if f < 1 or f > 32:
            continue
        span = (f - 1) * hop + N
        if span > 0x3fffffff:
            continue
        off = align_up(N * 4, 16)
        off = align_up(off + tw_count_split(log2m) * 8, 16)
        off = align_up(off + 8 * nh, 16)
        if mode == MODE_MEL:
            t = table_for(basis, rows_per_warp(f))
            off = align_up(off + len(t.w) * 4, 16)
            off = align_up(off + t.n_rows * 8, 16)                       # sizeof(MelRow) == 8
        if mode == MODE_STATS:
            off = align_up(off + (M + 1) * 4, 16)                        # bin frequencies
        off = align_up(off, 128)
        off += align_up(span * 4, 128) * nh
        off = align_up(off, 128)
        if mode in (MODE_MEL, MODE_STATS):
            xbytes = align_up(f * group_stride(M, f) * 8 + ((M + 16) * 4 if M < 128 else 0), 128)
        else:
            xbytes = align_up(f * (M + M // 32) * 8, 128)
        off += xbytes * nh
        if off <= smem_optin:
            return v, f, nh, off, xbytes
    return None


_tables = {}


def table_for(basis, H):
    key = (id(basis), H)
    if key not in _tables or _tables[key][0] is not basis:
        _tables[key] = (basis, row_table(basis, H))
    return _tables[key][1]


def first_refused_hop(n_fft, basis, smem_optin=H100_SMEM_OPTIN, mode=MODE_MEL):
    lo, hi = 1, 1 << 16                                                 # fits at lo, refused at hi (monotone)
    assert forward_choice(n_fft, hi, basis, smem_optin, mode) is None
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if forward_choice(n_fft, mid, basis, smem_optin, mode) else (lo, mid)
    return hi


def variant_runs(n_fft, basis, smem_optin=H100_SMEM_OPTIN, mode=MODE_MEL):
    """[(first hop, last hop, variant, FT)] of the instances `mode` selects, hop by hop, and the first refused
    hop."""
    stop = first_refused_hop(n_fft, basis, smem_optin, mode)
    runs = []
    for hop in range(1, stop):
        v, f = forward_choice(n_fft, hop, basis, smem_optin, mode)[:2]
        if runs and tuple(runs[-1][2:]) == (v, f):
            runs[-1][1] = hop
        else:
            runs.append([hop, hop, v, f])
    return [tuple(r) for r in runs], stop


# MODE_MEL at sr 22 050, 128 mels (default basis): (first hop, last hop, variant, FT) per size, then the first
# refused hop.  116 = two 8-warp halves.
H100_MEL_VARIANTS = {
    8: ([(1, 1825, 1, 32)], 1826),
    16: ([(1, 1823, 1, 32)], 1824),
    32: ([(1, 1818, 1, 32)], 1819),
    64: ([(1, 1779, 1, 32)], 1780),
    128: ([(1, 1701, 2, 32)], 1702),
    256: ([(1, 1518, 4, 32)], 1519),
    512: ([(1, 1221, 8, 32)], 1222),
    1024: ([(1, 608, 116, 16), (609, 626, 16, 32)], 627),
    2048: ([(1, 1001, 116, 8), (1002, 1111, 16, 16), (1112, 4717, 8, 8)], 4718),
    4096: ([(1, 618, 116, 4), (619, 1120, 16, 8), (1121, 8256, 8, 4)], 8257),
    8192: ([(1, 4928, 8, 2)], 4929),
}


# ------------------------------------------------------------------ run_mr / mr_block (spectrum_api.cu), mode 2
def mr_sizes():
    """Even n_fft of 12 ... 4096, not a power of two, whose half has no prime factor above 5 (pl.mr_covers)."""
    out = []
    for n in range(12, 4097, 2):
        if n & (n - 1) == 0:
            continue
        m = n // 2
        for q in (5, 3, 2):
            while m % q == 0:
                m //= q
        if m == 1:
            out.append(n)
    return out


def mr_tw_count(n_fft):
    count, sub = 0, 1
    for R in mr_factor(n_fft):
        if sub > 1:
            count += (R - 1) * sub
        sub *= R
    return max(count, 1)


def mr_table_bytes(L, tw_count, n_mels, mel_w_count):
    b = ((L + 3) & ~3) * 4 + ((tw_count + 1) & ~1) * 8 + ((L // 4 + 2) & ~1) * 8
    b += n_mels * 16 + ((mel_w_count + 3) & ~3) * 4                     # sizeof(MelBand) == 16
    return (b + 15) & ~15


def mr_choice(n_fft, basis, smem_optin=H100_SMEM_OPTIN):
    """(lanes per frame G, warps per block, shared-memory bytes) of run_mr in mel mode, or None (refused)."""
    M = n_fft // 2
    fpw = 2 if M <= 512 else 1
    tables = mr_table_bytes(n_fft, mr_tw_count(n_fft), basis.shape[0], sum(n for _, n in bands(basis)))
    per_warp = 2 * M * 8 * fpw
    budget = (smem_optin + 1024) // 2 - 1024
    w = 16
    while w > 1 and tables + w * per_warp > budget:
        w -= 1
    if tables + w * per_warp > smem_optin:
        return None
    return 32 // fpw, w, tables + w * per_warp


# ------------------------------------------------------------------ launch_dct (spectrum_api.cu)
def dct_choice(n_mels, n_mfcc, tiled, smem_optin=H100_SMEM_OPTIN):
    """"ks2" / "ks1" (dct_clamp4_kernel<KS>), "generic" (dct_generic_kernel) or "refused"."""
    KG = (n_mfcc + 7) // 8
    if KG > 16:
        return "refused"
    smem = (n_mels * 8 * KG + 2 * n_mels * 64) * 4
    if smem > smem_optin:
        return "refused" if tiled else "generic"
    return "ks2" if KG <= 10 and n_mels >= 8 * KG else "ks1"


# ================================================================== tests
def reachable_tiles():
    """{n_fft: sorted FT values} that MODE_MEL reaches on an H100 at any accepted hop (H100_MEL_VARIANTS)."""
    return {n: sorted({r[3] for r in runs}) for n, (runs, _) in H100_MEL_VARIANTS.items()}


def test_reachable_tiles():
    assert reachable_tiles() == {8: [32], 16: [32], 32: [32], 64: [32], 128: [32], 256: [32], 512: [32],
                                 1024: [16, 32], 2048: [8, 16], 4096: [4, 8], 8192: [2]}


@pytest.mark.parametrize("n_fft", SIZES)
def test_selection_table(n_fft):
    """The instance MODE_MEL selects at every hop up to the first refused one (sr 22 050, 128 mels)."""
    basis = mel_basis(22050, n_fft)
    assert variant_runs(n_fft, basis) == H100_MEL_VARIANTS[n_fft]
    runs, stop = H100_MEL_VARIANTS[n_fft]
    for first, last, v, f in runs:
        got = forward_choice(n_fft, last, basis)
        assert got[:2] == (v, f) and got[2] == (2 if v == 116 else 1) and got[3] <= H100_SMEM_OPTIN


def mel_grid(n_fft):
    """Mel configurations for one frame length: rates 8 ... 48 kHz, 1 ... 512 bands where the bins allow, band
    limits that leave empty rows, htk, every norm (spread over the grid)."""
    out = []
    combos = itertools.product([8000, 16000, 22050, 44100, 48000], [1, 2, 7, 13, 40, 80, 128, 256, 512],
                               [(0.0, None), (300.0, 4000.0), (2000.0, None)], [False, True])
    for i, (sr, n_mels, (fmin, fmax), htk) in enumerate(combos):
        if n_mels > 4 * (n_fft // 2 + 1) or (fmax is not None and fmax > sr / 2):
            continue
        if n_fft >= 1024 and i % 4 in (1, 2):                           # half of the grid for the long tables
            continue
        out.append(dict(sr=sr, n_mels=n_mels, fmin=fmin, fmax=fmax, htk=htk, norm=NORMS[i % len(NORMS)]))
    return out


def check_row_table(basis, n_fft, ft):
    """Every property of the MelRow table the fused kernel relies on, for one basis and one tile geometry."""
    M = n_fft // 2
    H = rows_per_warp(ft)
    rsm, G = max(H, 4), max(H, 4) // 4
    RS = 2 * group_stride(M, ft)
    assert RS >= M + 4 and RS % 32 == rsm % 32 and RS % 4 == 0
    t = row_table(basis, H)
    n_mels = basis.shape[0]
    assert t.n_rows % H == 0 and t.n_rows - n_mels < H
    assert (t.lo % 4 == 0).all() and (t.off % 4 == 0).all()
    assert t.lo.max() < 1 << 16 and t.quads.max() < 1 << 16
    assert len(t.w) == 4 * int(t.quads.sum())
    items = t.quads.reshape(-1, H)
    assert (items == items[:, :1]).all()                                 # one trip count per work item
    j = np.arange(t.n_rows) % H
    bank = t.lo % rsm == 4 * (j % G)
    bs = bands(basis) + [(0, 0)] * (t.n_rows - n_mels)
    b_lo = np.array([b[0] for b in bs])
    assert (bank | (b_lo - (b_lo - 4 * (j % G)) % rsm < 0)).all()     # the bank rule, but for the lowest rows
    # weights: the basis bit for bit inside the band, exact zeros around it, on every word a row reads
    dense = dense_rows(t, M, RS)
    got = dense[:n_mels, :M + 1].astype(np.float32)
    b32 = np.ascontiguousarray(basis, dtype=np.float32)
    nz = b32 != 0                                                        # the basis holds -0.0 too: a zero weight
    assert (got.view(np.uint32)[nz] == b32.view(np.uint32)[nz]).all() and not got[~nz].any()
    assert not dense[:n_mels, M + 1:].any() and not dense[n_mels:].any()
    # reads: words [lo, lo + 4 quads) of each frame the row's lanes own; the own frame's written words only
    end = t.lo + 4 * t.quads
    ok = written_words(M)
    assert end.max(initial=0) <= RS
    for m in range(t.n_rows):
        assert ok[t.lo[m]:end[m]].all(), (n_fft, ft, m, int(t.lo[m]), int(end[m]))
    # the last frame of a tile (FT - 1, the second frame of the last lane pair) ends inside the half's allocation
    xbytes = align_up(ft * group_stride(M, ft) * 8 + ((M + 16) * 4 if M < 128 else 0), 128)
    assert ((ft - 1) * RS + end.max(initial=0)) * 4 <= xbytes
    # the padded-row projection in float64 equals basis @ P, whatever the exchange words past bin M + 3 hold
    rng = np.random.default_rng(n_fft + ft + n_mels)
    P = rng.standard_normal((RS, 3)) ** 2
    P[M + 1:M + 4] = 0.0
    P[M + 4:] = rng.standard_normal((RS - M - 4, 3)) * 1e30
    proj = dense[:n_mels, :RS] @ P
    want = basis.astype(np.float64) @ P[:M + 1]
    np.testing.assert_allclose(proj, want, rtol=1e-12, atol=1e-300)
    return t


@pytest.mark.parametrize("n_fft", SIZES)
def test_row_table_invariants(n_fft):
    """check_row_table over the mel grid for every FT the size reaches, and for the last instance of each size the
    default basis (the table the benchmarks use)."""
    fts = reachable_tiles()[n_fft]
    configs = mel_grid(n_fft)
    assert len(configs) >= 40
    for kw in configs:
        basis = mel_basis(n_fft=n_fft, **kw)
        for ft in fts:
            check_row_table(basis, n_fft, ft)


def test_some_rows_read_past_the_nyquist_padding():
    """The invariant is not vacuous: reachable geometries read exchange words past bin M + 3, up to 12 words (n_fft
    8192, FT 2, htk, fmin 2 kHz), and rows of n_fft <= 32 read bins of the one-pass un-mix stores."""
    basis = mel_basis(8000, 8192, n_mels=256, fmin=2000.0, htk=True)
    t = row_table(basis, rows_per_warp(2))
    assert int((t.lo + 4 * t.quads).max()) - (4096 + 4) == 12


def test_a_read_of_an_unwritten_word_is_noticed():
    """written_words excludes the padding slots of the exchange layout and the group padding: a row table whose
    rows were moved by one quad past the band would read them."""
    M = 1024
    ok = written_words(M)
    pad_slots = [p for p in range(M + M // 32) if p % 33 == 32]
    assert pad_slots and not ok[2 * pad_slots[-1]] and not ok[2 * pad_slots[-1] + 1]
    assert not ok[2 * (M + M // 32)]
    assert written_words(16)[16 + 4 - 1] and not written_words(16)[2 * 16]


def test_mixed_radix_blocks():
    """All 96 mixed-radix sizes fit mr_kernel in mel mode with the default 128-band basis: G = 16 lanes per frame up
    to n_fft 1024, 32 above; two blocks per SM."""
    sizes = mr_sizes()
    assert len(sizes) == 96 and sizes[0] == 12 and sizes[-1] == 4050
    for n_fft in sizes:
        got = mr_choice(n_fft, mel_basis(22050, n_fft))
        assert got is not None, n_fft
        G, w, smem = got
        assert G == (16 if n_fft <= 1024 else 32) and 1 <= w <= 16 and smem <= (H100_SMEM_OPTIN + 1024) // 2 - 1024


@pytest.mark.parametrize("n_mels,n_mfcc,tiled,want", [
    (128, 20, True, "ks2"), (40, 13, True, "ks2"), (13, 20, True, "ks1"), (128, 100, True, "ks1"),
    (128, 128, True, "ks1"), (128, 129, True, "refused"), (382, 20, True, "ks2"), (383, 20, True, "refused"),
    (383, 20, False, "generic"), (512, 20, False, "generic"), (512, 20, True, "refused"), (13, 20, False, "ks1"),
])
def test_dct_selection(n_mels, n_mfcc, tiled, want):
    assert dct_choice(n_mels, n_mfcc, tiled) == want


# ------------------------------------------------------------------ sensitivity of the GPU test's comparison
def perturbed_bases(basis, n_fft, ft):
    """float64 bases of three subtly wrong kernels: weights rounded to 12 mantissa bits; the last quad of every
    padded row dropped; one row (the first non-empty one from the middle up) shifted up by one bin."""
    M = n_fft // 2
    b = basis.astype(np.float64)
    m, e = np.frexp(b)
    rounded = np.ldexp(np.round(m * 2.0 ** 12) / 2.0 ** 12, e)
    t = row_table(basis, rows_per_warp(ft))
    dense = dense_rows(t, M, 2 * group_stride(M, ft))
    for r in range(basis.shape[0]):
        q = int(t.quads[r])
        if q:
            dense[r, t.lo[r] + 4 * q - 4:t.lo[r] + 4 * q] = 0.0
    dropped = dense[:basis.shape[0], :M + 1]
    shifted = b.copy()
    r = basis.shape[0] // 2 + int(np.flatnonzero(b[basis.shape[0] // 2:].any(axis=1))[0])   # a non-empty row
    shifted[r] = np.roll(b[r], 1)
    return {"12-bit weights": rounded, "last quad dropped": dropped, "row shifted": shifted}


@pytest.mark.parametrize("n_fft", [64, 512, 2048, 8192])
def test_comparison_rejects_subtly_wrong_kernels(n_fft):
    """mel_close of the GPU test, fed float32-rounded float64 results of the wrong bases against the right one, on
    the GPU test's signals: every perturbation is rejected (the 12-bit weights by the norm-wise bound alone)."""
    import test_gpu_mel_front_end as G

    hop = n_fft // 4
    basis = mel_basis(22050, n_fft)
    ft = forward_choice(n_fft, hop, basis)[1]
    y = G.signals(3, G.n_samples(2 * ft + 1, n_fft, hop, True), n_fft, seed=n_fft)
    P = G.ref_power(y, n_fft, hop)
    ref = G.ref_mel(P, basis)
    G.mel_close(G.ref_mel(P, basis).astype(np.float32), ref, n_fft, "exact")     # the right basis passes
    for name, wrong in perturbed_bases(basis, n_fft, ft).items():
        got = G.ref_mel(P, wrong).astype(np.float32)
        with pytest.raises(AssertionError):
            G.mel_close(got, ref, n_fft, name)
        if name == "12-bit weights":                                    # the norm-wise bound alone rejects it
            with pytest.raises(AssertionError, match="u log2"):
                assert G.norm_ratio(got, ref) / np.log2(n_fft) <= G.C_MEL, f"{name}: u log2"
