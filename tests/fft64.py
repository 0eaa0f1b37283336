"""Float64 reference of the FFTContext transforms (libavcodec/fft.h:73-99) and the error measures the FFT / MDCT accuracy tests use.
TEST INFRASTRUCTURE: plain numpy, independent of both CPU oracles and of the kernels.

With N = 2^nbits and c(n, k) = cos(2 pi / N * (n + 1/2 + N/4) * (k + 1/2)):
  fft         forward X[k] = sum_j z[j] exp(-2 pi i jk / n); inverse with exp(+2 pi i jk / n) and no 1/n.  Natural order in and out.
  mdct_calc   out[k] =  scale * sum_{n < N}   x[n] c(n, k),   k < N/2
  imdct_calc  out[n] = -scale * sum_{k < N/2} X[k] c(n, k),   n < N
  imdct_half  imdct_calc restricted to n in [N/4, 3N/4)
Every phase is reduced to an integer residue modulo its period before it becomes an angle, so no argument exceeds 2 pi and the
basis is accurate to double rounding at every size.  The MDCT is a float64 matrix product up to MATRIX_MAX_BITS and an FFT-based
float64 evaluation above; tests/test_fft64_cpu.py pins the two forms to each other.  All functions work on the last axis, so a
(T, length) batch gives T transforms.
"""
import functools

import numpy as np

MATRIX_MAX_BITS = 12


def _cis(p, m):
    """exp(2 pi i p / m) for integer p, reduced modulo m first"""
    a = 2 * np.pi / m * (np.asarray(p, np.int64) % m)
    return np.cos(a) + 1j * np.sin(a)


def cplx(a):
    """interleaved float (..., 2n) -> complex128 (..., n)"""
    a = np.asarray(a, np.float64)
    return a[..., 0::2] + 1j * a[..., 1::2]


def interleave(z):
    """complex (..., n) -> interleaved float32 (..., 2n)"""
    z = np.asarray(z)
    out = np.empty(z.shape[:-1] + (2 * z.shape[-1],), np.float32)
    out[..., 0::2], out[..., 1::2] = z.real, z.imag
    return out


def fft(z, inverse):
    """complex (..., n) -> complex128 (..., n): the DFT of fft_permute + fft_calc"""
    z = np.asarray(z, np.complex128)
    return np.fft.ifft(z, axis=-1) * z.shape[-1] if inverse else np.fft.fft(z, axis=-1)


@functools.lru_cache(maxsize=2)
def _basis(nbits):
    """c(n, k) as an (N, N/2) float64 matrix"""
    N = 1 << nbits
    n, k = np.arange(N, dtype=np.int64)[:, None], np.arange(N // 2, dtype=np.int64)[None, :]
    return _cis((2 * n + 1 + N // 2) * (2 * k + 1), 4 * N).real


def mdct_matrix(x, nbits, scale):
    return scale * (np.asarray(x, np.float64) @ _basis(nbits))


def imdct_matrix(X, nbits, scale):
    return -scale * (np.asarray(X, np.float64) @ _basis(nbits).T)


def mdct_fft(x, nbits, scale):
    """out[k] = scale Re(exp(-2 pi i (n + n0)(k + 1/2) / N) summed over n), n0 = 1/2 + N/4, as one length-N complex FFT"""
    N = 1 << nbits
    x = np.asarray(x, np.float64)
    Y = np.fft.fft(x * _cis(-np.arange(N), 2 * N), axis=-1)[..., :N // 2]
    return scale * (_cis(-(1 + N // 2) * (2 * np.arange(N // 2) + 1), 4 * N) * Y).real


def imdct_fft(X, nbits, scale):
    """out[n] = -scale Re(sum over k of X[k] exp(-2 pi i (n + n0)(k + 1/2) / N)) as one zero-padded length-N complex FFT"""
    N = 1 << nbits
    X = np.asarray(X, np.float64)
    U = np.fft.fft(X * _cis(-(2 + N) * np.arange(N // 2), 4 * N), n=N, axis=-1)
    return -scale * (_cis(-(4 * np.arange(N) + 2 + N), 8 * N) * U).real


def mdct_calc(x, nbits, scale):
    return (mdct_matrix if nbits <= MATRIX_MAX_BITS else mdct_fft)(x, nbits, scale)


def imdct_calc(X, nbits, scale):
    return (imdct_matrix if nbits <= MATRIX_MAX_BITS else imdct_fft)(X, nbits, scale)


def imdct_half(X, nbits, scale):
    N = 1 << nbits
    return imdct_calc(X, nbits, scale)[..., N // 4:3 * N // 4]


OPS = {0: "imdct_half", 1: "imdct_calc", 2: "mdct_calc"}      # the op numbers of ff_mdct_batch_cuda


def mdct_sizes(op, nbits):
    """(input, output) length of one transform of ff_mdct_batch_cuda's op"""
    n = 1 << nbits
    return {0: (n // 2, n // 2), 1: (n // 2, n), 2: (n, n // 2)}[op]


def mdct_op(op, x, nbits, scale):
    return globals()[OPS[op]](x, nbits, scale)


def err(got, want):
    """norm-wise relative error ||got - want||_2 / ||want||_2 along the last axis (0 where both are zero)"""
    d = np.linalg.norm(np.asarray(got, np.complex128) - want, axis=-1)
    w = np.linalg.norm(np.asarray(want, np.complex128), axis=-1)
    return np.where(w > 0, d / np.where(w > 0, w, 1), np.where(d > 0, np.inf, 0.0))


def max_rel(got, want):
    """the north-star measure: max |got - want| / max |want| along the last axis (0 where both are zero)"""
    d = np.abs(np.asarray(got, np.complex128) - want).max(axis=-1)
    w = np.abs(np.asarray(want, np.complex128)).max(axis=-1)
    return np.where(w > 0, d / np.where(w > 0, w, 1), np.where(d > 0, np.inf, 0.0))
