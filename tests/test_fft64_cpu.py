"""CPU: pin the float64 reference of tests/fft64.py, which the GPU FFT / MDCT accuracy tests are measured against.

- Its two MDCT evaluations (matrix product, FFT-based) agree to float64 rounding, and the MDCT basis is orthogonal.
- The plain-C port (oracle/port/orc_fft.c: double core, float tables, float output) agrees with it to float output rounding.
- The unmodified reference's float FFTContext (oracle/_ref) agrees with it within REF_K * log2(N) * 2^-24 norm-wise.

Norm-wise error of the compiled reference against float64 on these tests' inputs (uniform(-1, 1) and Gaussian), largest over
both directions (FFT) or over the three ops and five scales (MDCT):
    FFT   nbits   2: 4.0e-8   3: 6.3e-8   4: 6.4e-8   5: 7.7e-8   6: 8.6e-8   7: 9.3e-8   8: 9.9e-8
                  9: 1.0e-7  10: 1.1e-7  11: 1.2e-7  12: 1.2e-7
    MDCT  nbits   4: 9.7e-8   5: 1.2e-7   6 .. 10: 1.2e-7   11: 1.3e-7   12: 1.3e-7   13: 1.4e-7   14: 1.4e-7
That is at most 0.41 * log2(N) * 2^-24 (log2(N) being the MDCT's own bits, not its inner FFT's) and 0.35 for the FFT, so
REF_K = 0.75 leaves a margin of 1.8.  The port stays within 1.1 * 2^-24.  test_gpu_fft_accuracy.py holds the GPU to the same
measure, against this reference on the same inputs.
"""
import numpy as np
import pytest

import fft64
from oracle.loader import ptr

ULP = 2.0 ** -24
REF_K = 0.75
PORT_BOUND = 2 * ULP
SCALES = [1.0, -1.0, 1.0 / 32768, 2.5, -1.0 / 7]


def inputs(rng, shape):
    return [rng.uniform(-1, 1, size=shape).astype(np.float32), rng.standard_normal(shape).astype(np.float32)]


@pytest.mark.parametrize("nbits", range(4, fft64.MATRIX_MAX_BITS + 1))
def test_mdct_forms_agree(nbits):
    """the FFT-based evaluation (used above MATRIX_MAX_BITS) against the matrix product, both ways, sign and scale included"""
    rng = np.random.default_rng(nbits)
    n = 1 << nbits
    x, X = rng.standard_normal((3, n)), rng.standard_normal((3, n // 2))
    for scale in SCALES:
        assert fft64.err(fft64.mdct_fft(x, nbits, scale), fft64.mdct_matrix(x, nbits, scale)).max() < 1e-14
        assert fft64.err(fft64.imdct_fft(X, nbits, scale), fft64.imdct_matrix(X, nbits, scale)).max() < 1e-14


@pytest.mark.parametrize("nbits", [4, 9, 14])
def test_mdct_basis_is_orthogonal(nbits):
    """mdct_calc(imdct_calc(X)) = -(N/2) X at scale 1: what lets the GPU tests read a weak tone back out of an IMDCT output"""
    n = 1 << nbits
    X = np.random.default_rng(nbits).standard_normal((2, n // 2))
    back = fft64.mdct_calc(fft64.imdct_calc(X, nbits, 1.0), nbits, 1.0)
    assert fft64.err(back, -(n / 2) * X).max() < 1e-13


def test_fft_known_answers():
    """impulse at j -> exp(-+2 pi i jk / n); a tone at bin k -> n at bin k; no 1/n on the inverse"""
    n = 64
    for j in (0, 1, 31, 32, 63):
        z = np.zeros(n, complex); z[j] = 1
        k = np.arange(n)
        assert np.abs(fft64.fft(z, 0) - fft64._cis(-j * k, n)).max() < 1e-15
        assert np.abs(fft64.fft(z, 1) - fft64._cis(j * k, n)).max() < 1e-15
    tone = np.exp(2j * np.pi * 5 * np.arange(n) / n)
    want = np.zeros(n, complex); want[5] = n
    assert np.abs(fft64.fft(tone, 0) - want).max() < 1e-12
    assert np.abs(fft64.fft(fft64.fft(tone, 0), 1) - n * tone).max() < 1e-10


def test_error_measures():
    w = np.array([[3.0, 4.0], [0.0, 0.0], [0.0, 0.0]])
    g = np.array([[3.0, 4.5], [0.0, 0.0], [0.0, 1e-30]])
    assert np.allclose(fft64.err(g, w), [0.1, 0.0, np.inf])
    assert np.allclose(fft64.max_rel(g, w), [0.125, 0.0, np.inf])


def _fft_case(oracle, nbits, inverse, z):
    a = z.copy()
    oracle.fft(nbits, inverse, ptr(a))
    return float(fft64.err(fft64.cplx(a), fft64.fft(fft64.cplx(z), inverse)))


def _mdct_case(oracle, op, nbits, scale, x):
    nout = fft64.mdct_sizes(op, nbits)[1]
    out = np.zeros(nout, np.float32)
    getattr(oracle, fft64.OPS[op])(nbits, scale, ptr(out), ptr(x.copy()))
    return float(fft64.err(out, fft64.mdct_op(op, x, nbits, scale)))


@pytest.mark.parametrize("nbits", range(2, 13))
@pytest.mark.parametrize("inverse", [0, 1])
def test_fft_port(orc, nbits, inverse):
    for z in inputs(np.random.default_rng(nbits * 2 + inverse), 2 << nbits):
        assert _fft_case(orc, nbits, inverse, z) < PORT_BOUND


@pytest.mark.parametrize("nbits", range(2, 13))
@pytest.mark.parametrize("inverse", [0, 1])
def test_fft_reference(refo, nbits, inverse):
    for z in inputs(np.random.default_rng(nbits * 2 + inverse), 2 << nbits):
        assert _fft_case(refo, nbits, inverse, z) < REF_K * nbits * ULP


@pytest.mark.parametrize("nbits", range(4, 15))
@pytest.mark.parametrize("scale", SCALES)
def test_mdct_port(orc, nbits, scale):
    rng = np.random.default_rng(nbits)
    for op in range(3):
        for x in inputs(rng, fft64.mdct_sizes(op, nbits)[0]):
            assert _mdct_case(orc, op, nbits, scale, x) < PORT_BOUND, (op, nbits, scale)


@pytest.mark.parametrize("nbits", range(4, 15))
@pytest.mark.parametrize("scale", SCALES)
def test_mdct_reference(refo, nbits, scale):
    rng = np.random.default_rng(nbits)
    for op in range(3):
        for x in inputs(rng, fft64.mdct_sizes(op, nbits)[0]):
            assert _mdct_case(refo, op, nbits, scale, x) < REF_K * nbits * ULP, (op, nbits, scale)
