"""CPU restatement of the algorithm of csrc/mr_kernel.cuh (host logic, no GPU): the radix schedule of `mr_factor`
(fives, threes, then eights and a four / two), Stockham autosort passes with the twiddle layout of the plan table,
the packed real-input trick and its un-mix, and the inverse through re/im-swapped forward passes — against
numpy.fft for every frame length the kernels serve.  The CUDA path itself is pinned by tests/test_gpu_parity.py."""
import numpy as np
import pytest


def mr_factor(n_fft):
    m, radices = n_fft // 2, []
    for q in (5, 3, 8):
        while m % q == 0:
            radices.append(q)
            m //= q
    if m % 4 == 0:
        radices.append(4)
        m //= 4
    if m % 2 == 0:
        radices.append(2)
        m //= 2
    assert m == 1
    return radices


def stockham(z, radices):
    """y[(i - k) R + k + q p] = sum_r x[i + r T] W_{pR}^{r k} W_R^{r q},  k = i mod p, T = M / R (one pass per radix)."""
    M, p = len(z), 1
    src = z.astype(np.complex128)
    for R in radices:
        T = M // R
        i = np.arange(T)
        k = i % p
        r = np.arange(R)
        u = src[i[None, :] + r[:, None] * T] * np.exp(-2j * np.pi * ((r[:, None] * k[None, :]) % (p * R)) / (p * R))
        v = np.exp(-2j * np.pi * np.outer(r, r) / R) @ u                 # v[q, i]
        dst = np.empty(M, dtype=np.complex128)
        dst[((i - k) * R + k)[None, :] + r[:, None] * p] = v
        src, p = dst, p * R
    return src


def mr_rfft(x):
    n_fft = len(x)
    M = n_fft // 2
    Z = stockham(0.5 * (x[0::2] + 1j * x[1::2]), mr_factor(n_fft))       # window * 1/2 folded in, as on the device
    k = np.arange(M // 2 + 1)
    A, B = Z[k], Z[(M - k) % M]
    e, o = A + np.conj(B), -1j * (A - np.conj(B))
    pp = np.exp(-2j * np.pi * k / n_fft) * o
    X = np.empty(M + 1, dtype=np.complex128)
    X[M - k] = np.conj(e - pp)
    X[k] = e + pp
    return X


def mr_irfft(X, n_fft):
    M = n_fft // 2
    k = np.arange(M // 2 + 1)
    xa, xb = X[k].copy(), X[M - k].copy()
    xa[0], xb[0] = xa[0].real, xb[0].real                                 # Im of DC / Nyquist ignored (irfft semantics)
    e, pq = xa + np.conj(xb), xa - np.conj(xb)
    o = np.exp(2j * np.pi * k / n_fft) * pq
    Zs = np.empty(M, dtype=np.complex128)
    Zs[(M - k) % M] = np.conj(e - 1j * o)
    Zs[k] = e + 1j * o
    swap = lambda z: z.imag + 1j * z.real
    r = stockham(swap(Zs), mr_factor(n_fft))
    out = np.empty(n_fft)
    out[0::2], out[1::2] = r.imag / n_fft, r.real / n_fft
    return out


def smooth_sizes():
    from librosa_b200 import _pipeline as pl

    return [n for n in range(12, 4097, 2) if pl.transform_path(n) == "mr"]


def test_schedule_and_transforms_for_every_size():
    rng = np.random.default_rng(0)
    sizes = smooth_sizes()
    assert len(sizes) == 96
    for n_fft in sizes:
        radices = mr_factor(n_fft)
        assert int(np.prod(radices)) == n_fft // 2 and len(radices) <= 12
        odd = [q for q in radices if q % 2]
        assert radices[:len(odd)] == odd                                  # odd radices first (bank rule of the p = 1 pass)
        x = rng.standard_normal(n_fft)
        X = np.fft.rfft(x)
        np.testing.assert_allclose(mr_rfft(x), X, rtol=0, atol=1e-11 * n_fft)
        Xi = X.copy()
        Xi[0] += 0.3j
        Xi[-1] -= 0.2j
        np.testing.assert_allclose(mr_irfft(Xi, n_fft), np.fft.irfft(Xi, n=n_fft), rtol=0, atol=1e-12)
