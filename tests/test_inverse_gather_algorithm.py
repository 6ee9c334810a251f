"""The scheduling of the power-of-two inverse (run_inverse in csrc/spectrum_api.cu, inv_kernel in csrc/inv_kernel.cuh)
restated in integer-indexed NumPy, in float64, on the CPU.  The windowed frames w * irfft(D) are taken as given, so
no FFT is involved: what is checked is the slot / piece / halo / round / carry scheme that turns frames into output
samples.  This file is the specification the kernel is read against.

Host side (run_inverse): the CTA variant (116 = 16 warps as two 8-warp halves, then 16 warps, then 8 warps; the first
whose tables, carry and exchange area fit the opt-in shared memory wins), its frames per round G, and the slot length
    frames_per_slot = max(ceil(total_frames / (sm_count * halves)), 4 G)   rounded up to a multiple of G.
Kernel side (inv_kernel): the (clip, frame) pairs of the batch form one sequence cut into slots; a slot is walked in
pieces, one per clip; a piece [fs, fe) clears the carry, starts its rounds at the first halo frame
fh = max(0, fs - (overlap - 1)) and owns the output positions [fs * hop, fe * hop) — to the end of the clip when it is
the clip's last piece.  A round holds ng <= G frames, gathers G + ceil(clen / hop) chunks of hop positions, emits the
owned chunks c_lo <= c < c_hi and keeps the rest as the next round's carry (clen = n_fft - hop floats, ping-pong).
After the last round the carry is flushed and the tail zero-filled.

Asserted over a seeded sweep of small geometries: the result equals a plain overlap-add (frames added in increasing
frame index) cropped to [start, start + out_len) and multiplied by inv_wss, bit for bit — the gather adds the same
terms in the same order; every output sample of every clip is written exactly once; the result does not depend on the
slot length.  The output starts as NaN and the carry that a round is about to fill starts as NaN, so a position or a
carry word the schedule forgets shows up.
"""
import numpy as np
import pytest

H100_SMEM_OPTIN = 232448          # cudaDevAttrMaxSharedMemoryPerBlockOptin of sm_90: 227 KB


# ------------------------------------------------------------------ host side: run_inverse
def align_up(x, a):
    return (x + a - 1) // a * a


def tw_count(log2m):
    """HostFftCfg::tw_count(): float2 twiddles of the register FFT of M = 2^log2m points."""
    M = 1 << log2m
    tpf = M // 32 if M >= 32 else 1
    ppt = M // tpf
    logp = int(np.log2(ppt))
    npass = 1 if ppt == 1 else (log2m + logp - 1) // logp
    count = 0
    for q in range(1, npass):
        radix = 1 << min(logp, log2m - q * logp)
        count += (radix - 1) << (q * logp)
    return count


def choose_variant(log2m, hop, smem_optin=H100_SMEM_OPTIN):
    """(variant, G, halves, shared-memory bytes) run_inverse picks for n_fft = 2^(log2m + 1), or None."""
    M = 1 << log2m
    N = 2 * M
    tpf = M // 32 if M >= 32 else 1
    variants = [116] if 9 <= log2m <= 11 else []
    variants += [16, 8] if log2m >= 10 else [min(16, tpf)]
    clen = max(N - hop, 0)
    for v in variants:
        nw, nh = (16, 2) if v == 116 else (v, 1)
        if nw * 32 % (tpf * nh):
            continue
        G = nw * 32 // nh // tpf
        if G < 1:
            continue
        off = align_up(N * 4, 16)
        off = align_up(off + tw_count(log2m) * 8, 16)
        off += align_up(2 * clen * 4, 16) * nh
        off = align_up(off, 128)
        off += align_up(G * (M + M // 32) * 8, 128) * nh
        if off <= smem_optin:
            return v, G, nh, off
    return None


def slot_length(total_frames, sm_count, halves, G):
    fps = -(-total_frames // (sm_count * halves))
    fps = max(fps, 4 * G)
    return align_up(fps, G)


def slot_count(total_frames, fps):
    return -(-total_frames // fps)


# ------------------------------------------------------------------ kernel side: inv_kernel
def inverse_gather(frames, hop, start, out_len, inv_wss, fps, G, halo=None, c_lo_off=0):
    """frames [clip, frame, n_fft] float64 (window already applied) -> (y [clip, out_len], writes [clip, out_len]).
    `halo`: frames re-transformed before a piece (the kernel's overlap - 1); `c_lo_off`: added to the first chunk a
    piece owns.  Other values than the defaults state a wrong kernel."""
    n_clips, n_frames, n_fft = frames.shape
    clen = max(n_fft - hop, 0)
    overlap = (n_fft + hop - 1) // hop
    halo = overlap - 1 if halo is None else halo
    y = np.full((n_clips, out_len), np.nan)
    writes = np.zeros((n_clips, out_len), dtype=np.int64)
    total = n_clips * n_frames

    def store(clip, o, val):
        assert len(np.unique(o)) == len(o)
        y[clip, o] = val * inv_wss[o]
        writes[clip, o] += 1

    for slot in range(slot_count(total, fps)):
        gpos, slot_end = slot * fps, min(total, (slot + 1) * fps)
        while gpos < slot_end:                                   # one piece per clip the slot touches
            clip, fs = divmod(gpos, n_frames)
            fe = min(n_frames, fs + (slot_end - gpos))
            gpos += fe - fs
            last_seg = fe == n_frames
            fh = max(0, fs - halo)
            emit_lo = fs * hop
            emit_hi = (1 << 62) if last_seg else fe * hop
            carry_cur, carry_nxt = np.zeros(clen), np.zeros(clen)
            fr0 = fh
            while fr0 < fe:
                ng = min(G, fe - fr0)
                emit_n = G * hop
                n_chunks = G + (clen + hop - 1) // hop
                o0 = fr0 * hop - start
                c_lo = max(0, (emit_lo - fr0 * hop + hop - 1) // hop + c_lo_off)
                c_hi = min(G, (emit_hi - fr0 * hop) // hop)
                item = np.arange(hop * n_chunks)
                c, i = item // hop, item % hop
                x = c * hop + i
                keep = x < emit_n + clen
                c, i, x = c[keep], i[keep], x[keep]
                q = np.where(i >= n_fft, -1, (n_fft - 1 - i) // hop)
                val = np.zeros(len(x))
                val[x < clen] = carry_cur[x[x < clen]]
                g_lo, g_hi = np.maximum(0, c - q), np.minimum(c, ng - 1)
                for g in range(ng):                              # increasing frame index: the reference's order
                    m = (g_lo <= g) & (g <= g_hi)
                    j = (c[m] - g) * hop + i[m]
                    assert ((0 <= j) & (j < n_fft)).all()
                    val[m] += frames[clip, fr0 + g, j]
                emit = x < emit_n
                o = o0 + x
                own = emit & (c >= c_lo) & (c < c_hi) & (o >= 0) & (o < out_len)
                store(clip, o[own], val[own])
                carry_nxt[:] = np.nan                            # every word is rewritten each round
                carry_nxt[x[~emit] - emit_n] = val[~emit]
                carry_cur, carry_nxt = carry_nxt, carry_cur
                fr0 += G
            if last_seg:
                u0 = fr0 * hop
                xs = np.arange(clen)
                o = u0 + xs - start
                ok = (o >= 0) & (o < out_len)
                store(clip, o[ok], carry_cur[xs[ok]])
                o = np.arange(max(0, u0 + clen - start), out_len)
                store(clip, o, np.zeros(len(o)))
    return y, writes


def overlap_add(frames, hop, start, out_len, inv_wss):
    n_clips, n_frames, n_fft = frames.shape
    buf = np.zeros((n_clips, max(n_fft + hop * (n_frames - 1), start + out_len)))
    for f in range(n_frames):
        buf[:, f * hop:f * hop + n_fft] += frames[:, f]
    return buf[:, start:start + out_len] * inv_wss


# ------------------------------------------------------------------ the sweep
def geometries(seed, count):
    """hop from 1 to above n_fft, G from 1 to 32, one- and two-frame clips, clips shorter than a slot, slot lengths
    from the host formula and every small multiple of G, start 0 and n_fft / 2, out_len below / at / above the
    span the frames cover."""
    rng = np.random.default_rng(seed)
    for k in range(count):
        n_fft = int(rng.choice([4, 8, 16, 32]))
        hop = int(rng.integers(1, n_fft + n_fft // 2 + 2))
        if k % 11 == 0:
            hop = int(rng.choice([1, n_fft // 4, n_fft // 2, n_fft - 1, n_fft, n_fft + 1]))
        G = int(rng.choice([1, 2, 4, 8, 16, 32]))
        n_frames = int(rng.choice([1, 2, int(rng.integers(3, 12)), int(rng.integers(12, 3 * G + 40))]))
        n_clips = int(rng.integers(1, 7)) if n_frames > 2 * G else int(rng.integers(1, 6 * G // n_frames + 8))
        total = n_clips * n_frames
        if k % 3 == 0:
            fps = slot_length(total, int(rng.integers(1, 9)), int(rng.integers(1, 3)), G)
        else:
            fps = G * int(rng.integers(1, max(2, total // G + 2)))
        start = n_fft // 2 if k % 2 else 0
        natural = n_fft + hop * (n_frames - 1) - 2 * start
        out_len = [natural, natural - int(rng.integers(1, n_fft + hop)), natural + int(rng.integers(1, 2 * n_fft + hop))][k % 5 % 3]
        yield dict(n_fft=n_fft, hop=hop, G=G, n_frames=n_frames, n_clips=n_clips, fps=fps, start=start,
                   out_len=max(1, out_len))


def run(geo, seed, **kw):
    rng = np.random.default_rng(seed)
    frames = rng.standard_normal((geo["n_clips"], geo["n_frames"], geo["n_fft"]))
    inv_wss = rng.uniform(0.5, 2.0, geo["out_len"])
    y, writes = inverse_gather(frames, geo["hop"], geo["start"], geo["out_len"], inv_wss, geo["fps"], geo["G"], **kw)
    return frames, inv_wss, y, writes


@pytest.mark.parametrize("seed", range(8))
def test_gather_equals_overlap_add_and_writes_every_sample_once(seed):
    for k, geo in enumerate(geometries(seed, 400)):
        frames, inv_wss, y, writes = run(geo, 1000 * seed + k)
        assert (writes == 1).all(), (geo, np.argwhere(writes != 1)[:4].tolist())
        np.testing.assert_array_equal(y, overlap_add(frames, geo["hop"], geo["start"], geo["out_len"], inv_wss), str(geo))
        # one slot for the whole batch, and the shortest slot the rounds allow: same bits
        for fps in (geo["n_clips"] * geo["n_frames"] + geo["G"], geo["G"]):
            if k % 4 == 0 and fps != geo["fps"]:
                y2, w2 = inverse_gather(frames, geo["hop"], geo["start"], geo["out_len"], inv_wss, fps, geo["G"])
                assert (w2 == 1).all(), (geo, fps)
                np.testing.assert_array_equal(y2, y, f"{geo} fps={fps}")


def test_every_cut_offset_inside_a_clip():
    """One geometry, every slot length from G up: the cuts visit every frame offset of the clips."""
    hop, G, n_fft, n_frames, n_clips = 3, 2, 16, 23, 5
    rng = np.random.default_rng(5)
    frames = rng.standard_normal((n_clips, n_frames, n_fft))
    out_len = n_fft + hop * (n_frames - 1) - n_fft // 2 + 9
    inv_wss = rng.uniform(0.5, 2.0, out_len)
    want = overlap_add(frames, hop, n_fft // 2, out_len, inv_wss)
    cuts = set()
    for fps in range(G, n_clips * n_frames + G, G):
        y, writes = inverse_gather(frames, hop, n_fft // 2, out_len, inv_wss, fps, G)
        assert (writes == 1).all(), fps
        np.testing.assert_array_equal(y, want)
        cuts |= {(s * fps) % n_frames for s in range(slot_count(n_clips * n_frames, fps))}
    assert cuts == set(range(n_frames))


@pytest.mark.parametrize("halo", [-1, +1])
def test_a_wrong_halo_is_noticed(halo):
    """The assertions above are not vacuous: with the halo one frame short, samples after a slot cut lose a frame.
    One frame too many changes nothing (the extra frame does not reach the piece), which is why the halo is
    overlap - 1 and not overlap."""
    wrong = same = 0
    for k, geo in enumerate(geometries(3, 300)):
        overlap = (geo["n_fft"] + geo["hop"] - 1) // geo["hop"]
        if overlap < 2:
            continue
        frames, inv_wss, y, writes = run(geo, k, halo=overlap - 1 + halo)
        assert (writes == 1).all()
        if np.array_equal(y, overlap_add(frames, geo["hop"], geo["start"], geo["out_len"], inv_wss)):
            same += 1
        else:
            wrong += 1
    assert (wrong > 50) if halo < 0 else (wrong == 0 and same > 50)


@pytest.mark.parametrize("off", [-1, +1])
def test_a_wrong_first_chunk_is_noticed(off):
    """A piece that starts its ownership one chunk late leaves samples unwritten.  One chunk early, two pieces write
    the same chunk, the intruder from a halo that is one frame short: on the device the rightful piece writes later
    and its value survives, so only the write count can tell."""
    counts = set()
    for k, geo in enumerate(geometries(4, 200)):
        counts |= set(np.unique(run(geo, k, c_lo_off=off)[3]).tolist())
    assert counts == ({1, 2} if off < 0 else {0, 1})


# ------------------------------------------------------------------ host side
def test_slot_length():
    rng = np.random.default_rng(0)
    for _ in range(2000):
        total = int(rng.integers(1, 10 ** int(rng.integers(1, 8))))
        sm, halves, G = int(rng.integers(1, 200)), int(rng.integers(1, 3)), 1 << int(rng.integers(0, 6))
        fps = slot_length(total, sm, halves, G)
        assert fps % G == 0 and fps >= 4 * G
        assert slot_count(total, fps) <= sm * halves or fps == 4 * G     # one slot per resident half, or the floor
        assert fps == 4 * G or (fps - G) * sm * halves < total           # no longer than it has to be


def test_variants_an_h100_reaches():
    """With 227 KB of opt-in shared memory: which (variant, G) serves which hop, for all eleven sizes.  No hop is
    refused.  The instances of inv_inst.cu that no hop reaches: 16 and 8 warps for n_fft 2048, 8 warps for 4096."""
    reached = {}
    for log2m in range(2, 13):
        n_fft = 2 << log2m
        for hop in range(1, 3 * n_fft + 1):
            got = choose_variant(log2m, hop)
            assert got is not None, (n_fft, hop)
            reached.setdefault(n_fft, {}).setdefault(got[:3], []).append(hop)
    spans = {n: {v: (min(h), max(h)) for v, h in d.items()} for n, d in reached.items()}
    for n_fft in (8, 16, 32, 64, 128, 256, 512):
        nw = max(1, min(16, n_fft // 64))
        assert spans[n_fft] == {(nw, 32, 1): (1, 3 * n_fft)}
    assert spans[1024] == {(116, 16, 2): (1, 3 * 1024)}
    assert spans[2048] == {(116, 8, 2): (1, 3 * 2048)}
    assert spans[4096] == {(16, 8, 1): (1, 47), (116, 4, 2): (48, 3 * 4096)}
    assert spans[8192] == {(8, 2, 1): (1, 4191), (16, 4, 1): (4192, 3 * 8192)}
    for n, d in reached.items():                                 # each variant serves one contiguous range of hops
        assert all(h == list(range(h[0], h[-1] + 1)) for h in d.values()), n
