"""CPU restatement of the algorithm of csrc/czt_kernel.cuh (host logic, no GPU): the chirp-z tables of `build_czt`
(csrc/plan.cu), two real frames packed into one complex transform, the product with FFT_P(h)/P, the inverse
transform as a re/im-swapped forward one, the un-mix of the two spectra through the mirror bin L - k, and the
inverse with its Hermitian extension (Im of DC and Nyquist dropped) — in float64, against scipy.fft.rfft / irfft
for every frame length the chirp-z kernels serve.  The CUDA path itself is pinned by tests/test_gpu_chirpz.py."""
import numpy as np
import scipy.fft as sf


def czt_sizes():
    """Frame lengths 3 ... 2047 served by the chirp-z kernels: neither a power of two nor mixed-radix."""
    from librosa_b200 import _pipeline as pl

    return [n for n in range(3, pl.MAX_CZT_N_FFT + 1) if pl.transform_path(n) == "czt"]


def czt_p(L):
    """Bluestein transform size: the smallest power of two >= 2L - 1, and at least 32 (one warp of the engine)."""
    P = 32
    while P < 2 * L - 1:
        P *= 2
    return P


def tables(L):
    """b[n] = exp(-i pi (n^2 mod 2L) / L), and FFT_P(h) / P with h[m] = conj b[|m|] wrapped to length P."""
    P = czt_p(L)
    n = np.arange(L)
    b = np.exp(-1j * np.pi * ((n * n) % (2 * L)) / L)
    h = np.zeros(P, dtype=np.complex128)
    h[0] = np.conj(b[0])
    h[1:L] = np.conj(b[1:])
    h[P - L + 1:] = np.conj(b[1:])[::-1]
    return P, b, sf.fft(h) / P


def swap(z):
    return z.imag + 1j * z.real


def fwd_pair(xa, xb, w):
    """Spectra (n_bins each) of the windowed real frames xa, xb through one complex chirp-z transform."""
    L = len(xa)
    P, b, hf = tables(L)
    a = np.zeros(P, dtype=np.complex128)
    a[:L] = (xa + 1j * xb) * (w * b)
    c = swap(sf.fft(swap(sf.fft(a) * hf)))          # IFFT_P(FFT_P(a) . FFT_P(h)) P, the 1/P folded into the table
    k = np.arange(L // 2 + 1)
    zk = c[k] * b[k]                                # Z[k]
    sgn = -1.0 if L & 1 else 1.0                    # b[L - k] = (-1)^L b[k]
    sk = np.where(k == 0, 1.0, sgn)                 # Z[L] is Z[0] itself
    zm = np.conj(c[np.where(k == 0, 0, L - k)]) * sk * np.conj(b[k])   # conj Z[L - k]
    return 0.5 * (zk + zm), (zk - zm) / 2j


def inv_pair(XA, XB, w, L):
    """Windowed irfft (length L) of two half spectra through one complex chirp-z transform."""
    P, b, hf = tables(L)
    nb = L // 2 + 1

    def hermitian(X):
        X = X.copy()
        X[0] = X[0].real                            # Im of DC is ignored, and of Nyquist for even L
        if L % 2 == 0:
            X[nb - 1] = X[nb - 1].real
        return np.concatenate([X, np.conj(X[1:L - nb + 1][::-1])])

    U = np.zeros(P, dtype=np.complex128)
    U[:L] = (hermitian(XA) + 1j * hermitian(XB)) * np.conj(b)
    c = swap(sf.fft(swap(sf.fft(U) * np.conj(hf))))
    u = c[:L] * np.conj(b) * w / L
    return u.real, u.imag


def test_chirpz_sizes_and_transform_sizes():
    sizes = czt_sizes()
    assert len(sizes) == 1962
    P = {czt_p(L) for L in sizes}
    assert sorted(P) == [1 << q for q in range(5, 13)]            # the eight instances of czt_inst.cu


def test_paired_forward_and_inverse_for_every_size():
    rng = np.random.default_rng(0)
    for L in czt_sizes():
        b = tables(L)[1]
        k = np.arange(1, L // 2 + 1)
        np.testing.assert_allclose(b[L - k], (-1) ** L * b[k], rtol=0, atol=1e-12)   # the un-mix mirror identity
        w = rng.uniform(0.1, 1.0, L)
        xa, xb = rng.standard_normal(L), 1e-3 * rng.standard_normal(L)      # 60 dB apart
        XA, XB = fwd_pair(xa, xb, w)
        RA, RB = sf.rfft(xa * w), sf.rfft(xb * w)
        scale = np.abs(RA).max()
        assert np.abs(XA - RA).max() <= 1e-13 * scale, L
        assert np.abs(XB - RB).max() <= 1e-13 * scale, L
        # the quiet frame keeps its own relative accuracy up to the loud partner's round-off
        assert np.linalg.norm(XB - RB) <= 1e-13 * np.linalg.norm(RA), L
        DA = RA + 1j * rng.standard_normal(RA.shape)                        # non-zero Im(DC), Im(Nyquist)
        DB = RB + 1e-3j * rng.standard_normal(RB.shape)
        ya, yb = inv_pair(DA, DB, w, L)
        wa, wb = sf.irfft(DA, n=L) * w, sf.irfft(DB, n=L) * w
        scale = np.abs(wa).max()
        assert np.abs(ya - wa).max() <= 1e-13 * scale, L
        assert np.abs(yb - wb).max() <= 1e-13 * scale, L


def test_gpu_sweep_covers_every_instance():
    """The size sweep of tests/test_gpu_chirpz.py reaches every chirp-z instance P at its smallest and largest
    frame length, and at an odd and an even one."""
    import test_gpu_chirpz as G

    sizes = czt_sizes()
    sweep = G.sweep_sizes()
    assert set(sweep) <= set(sizes) and len(sweep) == len(set(sweep))
    for P in sorted({czt_p(L) for L in sizes}):
        served = [L for L in sizes if czt_p(L) == P]
        swept = [L for L in sweep if czt_p(L) == P]
        assert min(served) in swept and max(served) in swept, P
        assert any(L % 2 for L in swept) and any(L % 2 == 0 for L in swept), P
    assert [L for L in sizes if L <= 256] == [L for L in sweep if L <= 256]   # all of P = 32 ... 512
