"""The host side and the algorithms of the feature kernels in csrc/feat_kernels.cuh restated in integer-indexed
NumPy, on the CPU: how b2l_spectral_contrast sizes contrast_kernel, how feature/stats.py reduces the octave bands,
which of the three contrast paths and which sort_keys<N> rung serves a band, the sorted-run merge of the fast path,
the block decomposition of frame_td_block_kernel and the rule that picks it, the hpss_kernel<NS> instance, and the
reflect index map of hpss_kernel.  This file is the specification the kernels are read against;
tests/test_gpu_feature_kernels.py runs them, with the case lists generated here.

Restated here:
    b2l_spectral_contrast (api.cu)  sort capacity cap = next power of two >= max(32, largest band count); per warp
                                    (Fp + cap) 4 bytes, Fp = (F + 3) & ~3; warps per block 8 -> 4 -> 2 -> 1, the first
                                    that fits the opt-in shared memory; refused when one warp does not fit
    contrast_kernel paths           kk = min(k, n);  kk <= 16 and n <= 512: sorted runs (lane l owns band bins l,
                                    l + 32, ...; sort_keys<2|4|8|16> by per = ceil(n / 32), none for per = 1), then
                                    the head walk (minima) and the s_top[-32 used] walk (maxima);  kk <= 16, n > 512:
                                    knock-out extraction;  kk > 16: bitonic sort of the band in shared memory
    b2l_frame_feature (api.cu)      frame_td_block_kernel when frame_length % hop == 0, R = frame_length / hop <= 64,
                                    n_clips <= 65 535 (clips on grid.y); frame_td_kernel otherwise
    frame_td_block_kernel           tiles of 64 frames; block g covers padded positions g hop - pad + [0, hop); a
                                    frame's count is the sum of its R blocks minus the crossing at its first position
                                    plus pad_first
    b2l_hpss (api.cu)               hpss_kernel<NS>, NS = 8 / 16 / 32 / 64 by max(win_harm, win_perc)
    reflect_index                   the np.pad "symmetric" extension, repeated for windows longer than the axis

The sizing tables are H100 constants (232 448 bytes of opt-in shared memory).  Last, the comparisons of the GPU test
must reject subtly wrong kernels simulated here on that test's own inputs.
"""
import numpy as np
import pytest

from test_inverse_gather_algorithm import H100_SMEM_OPTIN

# contrast_kernel: (warps per block, first F served with them) for one band over the whole row; then the first
# refused F.
CONTRAST_LADDER = [(8, 1), (4, 3169), (2, 6337), (1, 12673)]
CONTRAST_REFUSED_F = 25345
TD_FRAMES = 64
MAX_GRID_Y = 65535


# ------------------------------------------------------------------ contrast: sizing, bands, paths
def contrast_cap(counts):
    cap = 32
    while cap < max([1] + list(counts)):
        cap <<= 1
    return cap


def contrast_warps(F, counts, smem_optin=H100_SMEM_OPTIN):
    """Warps per block of contrast_kernel, 0 when refused."""
    per_warp = (((F + 3) & ~3) + contrast_cap(counts)) * 4
    nw = 8
    while nw > 1 and per_warp * nw > smem_optin:
        nw >>= 1
    return nw if per_warp * nw <= smem_optin else 0


def contrast_path(n, kk):
    """(path, sort_keys rung) of a band of n bins and tail length kk = min(k, n); rung 1 runs no network."""
    if kk <= 16 and n <= 512:
        per = (n + 31) >> 5
        rung = 16 if per > 8 else 8 if per > 4 else 4 if per > 2 else 2 if per > 1 else 1
        return "runs", rung
    return ("knockout" if kk <= 16 else "bitonic"), 0


def contrast_cases():
    """(n, k) pairs that reach every path x rung, each at both sides of its rung and path boundaries."""
    cases = []
    for n in (1, 2, 31, 32, 33, 64, 65, 128, 129, 256, 257, 512, 513, 1000):
        for k in (1, 2, 16, 17, 40):
            if k <= max(n, 1) or k in (2, 17):
                cases.append((n, k))
    return cases


def test_contrast_ladder():
    """The F at which each warps-per-block rung starts, and the first refused F (one band over the whole row)."""
    got, prev = [], None
    for F in range(1, 30000):
        nw = contrast_warps(F, [F])
        if nw != prev:
            got.append((nw, F))
            prev = nw
    assert got[:-1] == CONTRAST_LADDER and got[-1] == (0, CONTRAST_REFUSED_F)
    # a band list whose longest band is short keeps 8 warps far longer: the capacity follows the longest band
    assert contrast_warps(6000, [200, 1000]) == 8 and contrast_cap([0]) == 32 and contrast_cap([33]) == 64


def test_contrast_path_table():
    """Every (n, kk) pair up to n = 1024: the rung boundaries n = 32/33, 64/65, 128/129, 256/257, 512/513 and the path
    boundary kk = 16/17, and the generated case list reaches every path x rung."""
    for n in range(0, 1025):
        for kk in range(0, min(n, 40) + 1):
            path, rung = contrast_path(n, kk)
            if kk > 16:
                assert path == "bitonic"
            elif n > 512:
                assert path == "knockout"
            else:
                assert path == "runs" and rung == {0: 1, 1: 1, 2: 2, 3: 4, 4: 4}.get(-(-n // 32), 8 if n <= 256 else 16)
    edges = {(32, 33): (1, 2), (64, 65): (2, 4), (128, 129): (4, 8), (256, 257): (8, 16)}
    for (a, b), (ra, rb) in edges.items():
        assert contrast_path(a, 1) == ("runs", ra) and contrast_path(b, 1) == ("runs", rb)
    assert contrast_path(512, 16) == ("runs", 16) and contrast_path(513, 16)[0] == "knockout"
    assert contrast_path(100, 17)[0] == "bitonic"
    reached = {contrast_path(n, min(k, n)) for n, k in contrast_cases()}
    assert reached == {("runs", r) for r in (1, 2, 4, 8, 16)} | {("knockout", 0), ("bitonic", 0)}


def librosa_band_masks(freq, sr, fmin, n_bands, quantile):
    """librosa's spectral_contrast masks (feature/spectral.py:483-499), as the selected bins and the tail length."""
    octa = np.zeros(n_bands + 2)
    octa[1:] = fmin * (2.0 ** np.arange(0, n_bands + 1))
    out = []
    for k, (f_low, f_high) in enumerate(zip(octa[:-1], octa[1:])):
        current_band = np.logical_and(freq >= f_low, freq <= f_high)
        idx = np.flatnonzero(current_band)
        if k > 0:
            current_band[idx[0] - 1] = True
        if k == n_bands:
            current_band[idx[-1] + 1:] = True
        rows = np.flatnonzero(current_band)
        if k < n_bands:
            rows = rows[:-1]
        out.append((rows, int(np.maximum(np.rint(quantile * np.sum(current_band)), 1))))
    return out, octa


@pytest.mark.parametrize("n_fft, sr, fmin, n_bands, quantile, freq", [
    (64, 22050, 200.0, 6, 0.02, None), (2048, 22050, 200.0, 6, 0.02, None), (1024, 16000, 100.0, 4, 0.25, None),
    (400, 16000, 200.0, 5, 0.02, None), (32768, 44100, 1.3, 15, 0.1, None), (4096, 44100, 20.0, 10, 0.5, None),
    (2048, 22050, 200.0, 6, 0.02, "log")])
def test_contrast_band_reduction(n_fft, sr, fmin, n_bands, quantile, freq):
    """feature/stats.py's (lo, count, k) per band equals librosa's masks: contiguous rows lo .. lo + count - 1, the
    last band to Nyquist, the empty band 0 at n_fft 64 (NaN, like np.mean of an empty slice), 15 bands, a custom
    increasing freq."""
    from librosa_b200.feature.stats import _contrast_bands

    F = n_fft // 2 + 1
    f = np.fft.rfftfreq(n_fft, 1.0 / sr) if freq is None else np.geomspace(10.0, sr / 2, F)
    masks, octa = librosa_band_masks(f, sr, fmin, n_bands, quantile)
    bands = _contrast_bands(f, octa, quantile)
    assert len(bands) == n_bands + 1
    for (rows, q), (lo, count, k) in zip(masks, bands):
        assert np.array_equal(rows, np.arange(lo, lo + count)) and k == q
    assert bands[-1][0] + bands[-1][1] == F                    # the last band runs to Nyquist
    if n_fft == 64:
        assert bands[0][1] == 0                                # 200 Hz lies above the first bin spacing: empty
        assert np.isnan(np.mean(np.zeros((0,))))


def float_keys(x):
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return np.where(u & 0x80000000, ~u & 0xffffffff, u | 0x80000000).astype(np.uint64)


def runs_extract(vals, k, tail_off=0):
    """The fast path's merge on one band (float32 vals): per-lane sorted runs, the k smallest off the heads and the k
    largest off the tails (s_top[-32 (used + tail_off)]), summed in float32 in extraction order.  Returns
    (valley, peak) as float32 means; tail_off = 1 is the walk one entry too low."""
    n = len(vals)
    kk = min(k, n)
    runs = [np.sort(float_keys(vals[l::32])) for l in range(32)]
    key_to_val = dict(zip(float_keys(vals).tolist(), np.asarray(vals, np.float32).tolist()))
    big, small = np.uint64(0xffffffff), np.uint64(0)

    def walk(pick, pos, cand):
        acc = np.float32(0.0)
        used = [0] * 32
        for _ in range(kk):
            c = [cand(l, used[l]) for l in range(32)]
            live = [l for l in range(32) if used[l] < len(runs[l])]
            win = pick(c)
            owners = [l for l in live if c[l] == win]
            if not owners:
                break
            used[owners[0]] += 1
            acc = np.float32(acc + np.float32(key_to_val.get(int(win), 0.0)))
        return acc

    lo = walk(min, 0, lambda l, h: runs[l][h] if h < len(runs[l]) else big)

    def top(l, used):
        i = len(runs[l]) - 1 - used - (tail_off if used else 0)
        return runs[l][i] if used < len(runs[l]) and 0 <= i < len(runs[l]) else small
    hi = walk(max, 0, top)
    return np.float32(lo / np.float32(kk)), np.float32(hi / np.float32(kk))


def layout(kind, n, k, rng):
    """A band of n magnitudes: random, all equal, mostly zeros, duplicates, or the k smallest and the k largest all in
    one lane (lane 0, lane 31, or the lane of the last bin)."""
    if kind == "equal":
        return np.full(n, 0.75, np.float32)
    if kind == "zeros":
        v = rng.uniform(0.0, 1.0, n).astype(np.float32)
        v[rng.random(n) < 0.7] = 0.0
        return v
    if kind == "dups":
        return (rng.integers(0, 4, n) * 0.5).astype(np.float32)
    v = rng.uniform(1.0, 2.0, n).astype(np.float32)
    if kind == "random":
        return v
    lane = {"lane0": 0, "lane31": 31, "lastlane": (n - 1) % 32}[kind]
    slots = np.arange(lane, n, 32)
    if slots.size == 0:
        return v
    m = min(k, slots.size)
    half = max(1, slots.size // 2) if slots.size > 1 else 1
    lo_slots, hi_slots = slots[:min(m, half)], slots[slots.size - min(m, slots.size - min(m, half)):]
    v[lo_slots] = rng.uniform(0.0, 0.5, lo_slots.size)
    if slots.size > 1:
        v[hi_slots] = rng.uniform(3.0, 4.0, hi_slots.size)
    return v


KINDS = ["random", "equal", "zeros", "dups", "lane0", "lane31", "lastlane"]


@pytest.mark.parametrize("n", [1, 5, 31, 32, 33, 64, 65, 100, 128, 129, 256, 257, 300, 512])
def test_contrast_run_merge(n):
    """The run merge equals the np.sort tails on adversarial layouts (n < 32 leaves lanes empty)."""
    rng = np.random.default_rng(n)
    for k in (1, 3, 9, 16):
        for kind in KINDS:
            v = layout(kind, n, k, rng)
            kk = min(k, n)
            s = np.sort(v)
            lo, hi = runs_extract(v, k)
            assert np.isclose(lo, s[:kk].astype(np.float64).mean(), rtol=kk * 2.0 ** -23, atol=0)
            assert np.isclose(hi, s[n - kk:].astype(np.float64).mean(), rtol=kk * 2.0 ** -23, atol=0)


# ------------------------------------------------------------------ time-domain framings
def td_choice(L, hop, n_clips, T):
    """True: frame_td_block_kernel; False: frame_td_kernel."""
    tiles = (T + TD_FRAMES - 1) // TD_FRAMES
    return L % hop == 0 and L // hop <= 64 and n_clips <= MAX_GRID_Y and tiles <= 0x7fffffff


def load_padded(y, j, mode, pad):
    """load_padded (common.cuh) at any integer positions j (array) of the float32 signal y."""
    n = len(y)
    j = np.asarray(j, np.int64)
    inside = (j >= 0) & (j < n)
    out = np.zeros(j.shape, np.float32)
    out[inside] = y[j[inside]]
    o = ~inside
    if mode == "edge":
        out[o] = np.where(j[o] < 0, y[0], y[-1])
    elif mode == "reflect":
        if n == 1:
            out[o] = y[0]
        else:
            m = np.mod(j[o], 2 * (n - 1))
            out[o] = y[np.where(m >= n, 2 * (n - 1) - m, m)]
    elif mode == "symmetric":
        m = np.mod(j[o], 2 * n)
        out[o] = y[np.where(m >= n, 2 * n - 1 - m, m)]
    elif mode == "linear_ramp":
        d = np.where(j[o] < 0, -j[o], j[o] - (n - 1))
        edge = np.where(j[o] < 0, y[0], y[-1]).astype(np.float64)
        i = pad - d
        out[o] = np.where(i <= 0, 0.0, i * (edge / max(pad, 1))).astype(np.float32)     # pad 0: no ramp
    return out


def sign_class(x, threshold, zero_pos):
    x = np.where(np.abs(x) <= threshold, np.float32(0.0), x)
    return (x < 0).astype(np.int64) if zero_pos else np.sign(x).astype(np.int64)


def block_counts(y, L, hop, center, mode, threshold=0.0, zero_pos=1, pad_first=0, subtract_first=True):
    """frame_td_block_kernel's zero-crossing counts in integers: per 64-frame tile, the 64 + R - 1 blocks (sum of
    crossings at positions p0 .. p0 + hop - 1, each against the sample before it, and the crossing at p0), then every
    frame = its R block sums - first + pad_first."""
    n = len(y)
    R = L // hop
    pad = L // 2 if center else 0
    T = 1 + (n + 2 * pad - L) // hop
    out = np.empty(T, np.int64)
    for t0 in range(0, T, TD_FRAMES):
        g = t0 + np.arange(TD_FRAMES + R - 1)
        p0 = g * hop - pad
        pos = p0[:, None] + np.arange(-1, hop)[None, :]
        c = sign_class(load_padded(y, pos, mode, pad), threshold, zero_pos)
        cross = c[:, 1:] != c[:, :-1]
        val, first = cross.sum(axis=1), cross[:, 0].astype(np.int64)
        f = np.arange(min(TD_FRAMES, T - t0))
        sums = np.array([val[i:i + R].sum() for i in f])
        out[t0 + f] = sums - (first[f] if subtract_first else 0) + int(pad_first != 0)
    return out


def direct_counts(y, L, hop, center, mode, threshold=0.0, zero_pos=1, pad_first=0):
    """zero crossings per frame of np.pad(y) (librosa's framing), positions 1 .. L - 1, plus pad_first."""
    yp = np.pad(y.astype(np.float64), L // 2, mode=mode) if center else y.astype(np.float64)
    fr = np.lib.stride_tricks.sliding_window_view(yp, L)[::hop]
    c = sign_class(fr.astype(np.float32), threshold, zero_pos)
    return (c[:, 1:] != c[:, :-1]).sum(axis=1) + int(pad_first != 0)


@pytest.mark.parametrize("hop", [1, 3, 4, 128, 129, 512])
@pytest.mark.parametrize("center, mode", [(False, "constant")] + [(True, m) for m in
                                          ("constant", "edge", "reflect", "symmetric", "linear_ramp")])
def test_td_block_decomposition(hop, center, mode):
    """For every R in 1 .. 64 (and 65, which takes frame_td_kernel) and T mod 64 in {0, 1, 63}: the block sums minus
    first[f] plus pad_first equal the direct count of every frame, exactly."""
    rng = np.random.default_rng(hop)
    Rs = list(range(1, 65)) if hop < 128 else [1, 2, 3, 4, 7, 8, 16, 31, 63, 64]
    for R in Rs + [65]:
        L = R * hop
        assert td_choice(L, hop, 1, 64) == (R <= 64)
        if R > 64:
            continue
        for T in (64, 65, 63):
            n = (T - 1) * hop + ((L - 2 * (L // 2)) if center else L) + rng.integers(0, hop)
            y = rng.integers(-2, 3, n).astype(np.float32) * np.float32(0.5)
            y[rng.random(n) < 0.5] += np.float32(0.25)
            for pf in (0, 1):
                got = block_counts(y, L, hop, center, mode, pad_first=pf, zero_pos=pf)
                ref = direct_counts(y, L, hop, center, mode, pad_first=pf, zero_pos=pf)
                assert len(got) == T and np.array_equal(got, ref), (R, T, pf)


def test_td_kernel_choice():
    assert td_choice(2048, 512, 1, 100) and td_choice(64 * 7, 7, 65535, 1)
    assert not td_choice(65 * 7, 7, 1, 100)                   # R = 65
    assert not td_choice(1000, 300, 1, 100)                   # not a multiple
    assert not td_choice(2048, 512, 65536, 1)                 # clips beyond grid.y: the per-frame kernel


# ------------------------------------------------------------------ hpss
def hpss_instance(win_harm, win_perc):
    w = max(win_harm, win_perc)
    return 8 if w <= 8 else 16 if w <= 16 else 32 if w <= 32 else 64


def reflect_index(i, n):
    while i < 0 or i >= n:
        i = -i - 1 if i < 0 else 2 * n - i - 1
    return i


def test_hpss_instance():
    assert [hpss_instance(w, 1) for w in (1, 8, 9, 16, 17, 32, 33, 64)] == [8, 8, 16, 16, 32, 32, 64, 64]
    assert hpss_instance(31, 31) == 32 and hpss_instance(3, 33) == 64


def test_reflect_index_is_symmetric_pad():
    """For every n <= 70 and w <= 64 the window of element t (t - w // 2 + j, j < w) through reflect_index is the
    np.pad(..., "symmetric") extension."""
    for n in range(1, 71):
        for w in range(1, 65):
            xp = np.pad(np.arange(n), (w // 2, w - 1 - w // 2), mode="symmetric")
            for t in range(n):
                assert [reflect_index(t - w // 2 + j, n) for j in range(w)] == list(xp[t:t + w])


def test_scipy_reflect_median_where_defined():
    """A pinned fact about the reference's median filter: scipy.ndimage.median_filter(mode="reflect") equals the
    median over the np.pad symmetric extension wherever the half-window w // 2 fits in the axis; where it does not,
    scipy returns values that are not in the input (uninitialised memory), so the GPU test's reference is the
    np.pad form, and the kernel's answer there is intended.  maximum_filter1d (pcen / onset max_size) agrees
    everywhere."""
    import scipy.ndimage as nd

    rng = np.random.default_rng(0)
    for n in range(1, 40):
        for w in range(1, 65):
            x = rng.standard_normal(n)
            xp = np.pad(x, (w // 2, w - 1 - w // 2), mode="symmetric")
            win = np.lib.stride_tricks.sliding_window_view(xp, w)
            assert np.array_equal(nd.maximum_filter1d(x, size=w, mode="reflect"), win.max(axis=-1))
            if w // 2 <= n:
                assert np.array_equal(nd.median_filter(x, size=w, mode="reflect"), np.sort(win, -1)[:, w // 2])


# ------------------------------------------------------------------ the GPU file's comparisons reject wrong kernels
def test_comparisons_reject_wrong_kernels():
    """The GPU test's checks, fed the results of simulated wrong kernels on its own kinds of input: the max-tail walk
    one entry off, a tail mean over k - 1 values, first[f] not subtracted, the even-window median rank w / 2 - 1,
    pcen's default zi taken as 0."""
    import test_gpu_feature_kernels as G

    rng = np.random.default_rng(11)
    # contrast: fast path, maxima all in one lane
    n, k = 100, 5
    S = np.stack([layout(kd, n, k, rng) for kd in ("lane0", "lane31", "lastlane", "random")])
    bands = [(0, n, k)]
    right = np.array([runs_extract(r, k) for r in S])
    G.contrast_close(right[None, :, 1], right[None, :, 0], S, bands, "exact")
    wrong = np.array([runs_extract(r, k, tail_off=1) for r in S])
    assert (wrong[:, 1] != right[:, 1]).any()
    with pytest.raises(AssertionError):
        G.contrast_close(wrong[None, :, 1], right[None, :, 0], S, bands, "tail walk off by one")
    s = np.sort(S, axis=-1).astype(np.float64)
    km1 = (s[:, :k].sum(-1) / (k - 1)).astype(np.float32)
    with pytest.raises(AssertionError):
        G.contrast_close(right[None, :, 1], km1[None], S, bands, "mean over k - 1")
    # zero crossings: first[f] not subtracted
    y = rng.integers(-2, 3, 5000).astype(np.float32)
    got = block_counts(y, 2048, 512, True, "edge", subtract_first=False)
    ref = G.ref_crossings(y[None], 2048, 512, True, "edge", 0.0, 1, 0)[0]
    assert np.array_equal(block_counts(y, 2048, 512, True, "edge"), ref) and not np.array_equal(got, ref)
    # hpss: even window, rank w / 2 - 1
    M, _ = G.hpss_input(1, 30, 20, seed=3)
    mh, mp = G.hpss_ref(M, 8, 6, (1.0, 1.0), 2.0, rank_h=3, rank_p=2)
    G.hpss_close(G.hpss_ref(M, 8, 6, (1.0, 1.0), 2.0), M, None, 8, 6, (1.0, 1.0), 2.0, True, "exact")
    with pytest.raises(AssertionError):
        G.hpss_close((mh.astype(np.float32), mp.astype(np.float32)), M, None, 8, 6, (1.0, 1.0), 2.0, True, "rank")
    # pcen: zi = 0 instead of 1 - b
    S = G.pcen_input(1, 33, 65, seed=1)
    ok, _ = G.pcen_ref(S, 0.98, 2.0, 0.5, 1e-6, 0.025, 1)
    G.pcen_close(ok.astype(np.float32), S, 0.98, 2.0, 0.5, 1e-6, 0.025, 1, "exact")
    bad, _ = G.pcen_ref(S, 0.98, 2.0, 0.5, 1e-6, 0.025, 1, zi=np.zeros((1, 33)))
    with pytest.raises(AssertionError):
        G.pcen_close(bad.astype(np.float32), S, 0.98, 2.0, 0.5, 1e-6, 0.025, 1, "zi = 0")
